// mde_solver.cu -- device-resident projected L-BFGS (the MDE.embed solve loop).
//
// Replaces optim.lbfgs (pymde/optim.py:69-184) driving LBFGS.step (pymde/lbfgs.py:390-590),
// _strong_wolfe (pymde/lbfgs.py:44-253), the value_and_grad closure (pymde/optim.py:100-105)
// and the per-iteration callback/statistics (pymde/optim.py:94-96,139-173).
//
// Design:
//  * every vector (X, x_init, d, g, g_prev, the S/Y history ring) and every scalar (loss,
//    g.d, Wolfe bracket, Gram matrix of the history, statistics) lives in HBM; the host
//    only enqueues kernels and reads one 32-byte status word per line-search trial
//    (mode 0) or per batch of iterations (mode 1, CUDA graph with a device-side while loop);
//  * the two-loop recursion is done on the (2h+1)^2 Gram matrix ("vector-free" L-BFGS):
//    ONE pass computes all 5h+4 dot products and writes the new (s, y) pair, ONE pass forms
//    d = cg*g + sum cs_j s_j + cy_j y_j (and snapshots g_prev, x_init, g.d, |d|, |X|).
//    The reference does 4h n*m-sized passes and 2h host syncs per iteration;
//  * reductions are two-stage with a fixed order (per-block partials -> one-block finalize),
//    so scalars are bit-reproducible for a given launch shape -- required for the replicated
//    multi-GPU solve where every rank must take the same Wolfe decisions;
//  * reference quirk kept on purpose (SURVEY section 7.5): the gradient seen by iteration k+1 is
//    the one left by the LAST trial of iteration k's line search, the loss is the ACCEPTED
//    trial's loss.
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <new>

#include "mde_common.cuh"
#include "mde_logic.h"
#include "mde_project.cuh"

struct mde_edges;
namespace mde {
int distortion_fused(const mde_edges* e, const float* X, int m, float* grad, int* nblocks, cudaStream_t st);
int distortion_fused_flag(const mde_edges* e, const float* X, int m, float* grad, int* nblocks,
                          const int* flag, cudaStream_t st);
const double* loss_partials_ptr(const mde_edges* e);
int64_t edges_n(const mde_edges* e);
int64_t edges_p_total(const mde_edges* e);
}  // namespace mde

using namespace mde;

namespace {

constexpr int kVecThreads = 256;
constexpr int kVecBlocks = kNumSMs * 2;
constexpr int kPairsPerSlice = 10;  // the default history (memory_size = 10, optim.py:110) fits ONE slice: one wave
constexpr int kDotsPerSlice = 4 + 5 * kPairsPerSlice;  // 54
constexpr int kMaxSlices = (kMaxMemory + kPairsPerSlice - 1) / kPairsPerSlice;  // 4
constexpr int kHeadAcc = kDotsPerSlice + 12;  // step_head_kernel: + g.d, g.g, |g|_1, column sums of g and X (+ pad): fp32 accumulators
constexpr int kHeadCols = kHeadAcc + 6;       // columns of a partial row: + loss, (g.d, d.d, X.X, max|d|) of the vec kernel, pad (even)
constexpr int kStatusInts = 12;
enum { PH_DIR = 0, PH_TRIAL = 1, PH_FRESH = 2, PH_MAT = 3 };  // mode 2: phase of a step

struct alignas(16) HeadDesc {  // what every block of the next head kernel needs, in 64 bytes (4 broadcast loads)
  int pend, phase, count, n_iter;
  int cand; float t_cur, t_last; int pad;
  unsigned char order[32];   // logical -> physical slot of the stored pairs (kMaxMemory <= 32)
};

struct SolverState {
  // ---- status word (first kStatusInts ints, copied to the host) ----
  int active;      // kernels exit early when 0
  int converged;   // residual test fired (optim.py:165)
  int iter;        // completed iterations
  int error;       // MDE_E_NAN when the reference would raise SolverError
  int need_fresh;  // lbfgs n_iter == 0: evaluate at X before the direction update
  int ls_active;   // line search wants another trial
  int stop_after;  // residual <= eps seen at the start of this iteration
  int pad0;        // low word of func_evals
  // ---- mode 2 (flat step graph) ----
  int paused;      // stopped at iter_limit; mde_solver_run resumes it
  int phase;       // what the next step does (PH_*)
  int iter_limit;  // pause when `iter` reaches it
  int pend;        // late-epilogue steps: 1 = the previous step executed phase `phase`, its bookkeeping is pending
  int g_dir;       // gates of the next step, written by the step epilogue: direction kernels run
  int g_eval;      //   closure evaluation (scatter kernel, tangent projection, dots) runs
  int g_mat;       //   the axpy materialises the ACCEPTED point (no evaluation follows)
  int g_proj;      //   the iterate moved: retraction kernels run
  // ---- scalars ----
  double eps;
  double loss;     // f at the current iterate (cached loss, lbfgs.py:418-426,550)
  double gg, g1;   // ||g||^2 and ||g||_1 of the gradient buffer
  float gtd;       // g.d
  float dmax;      // max |d|
  double dd, xx;   // ||d||^2, ||X||^2 at iteration start
  unsigned int tickets[4];   // last-block-done counters of the fused vector+scalar kernels
  float mu_x[4], mu_d[4];  // column means of x_init and d (Centered, m in {1,2,4}: fused into the trial axpy)
  double t_last;   // state["t"]
  double t_eval;   // step of the most recent trial evaluation
  long long func_evals;
  int max_stats;
  int world;
  double *avg, *resid, *pct, *steplen;
  // ---- late-epilogue steps ----
  double t_cur;                      // step length the current step's vec kernel applies (t0 / ls.t / ls.t_accept)
  double cs_g[4], cs_d[4];           // column sums of g_prev and d (tracked through the two-loop coefficients)
  double cs_S[kSlots][4], cs_Y[kSlots][4];  // ... and of the stored pairs
  HeadDesc hd;                       // written by init / the head kernel's epilogue for the NEXT head kernel
  unsigned long long dbg[12];        // globaltimer stamps of the last head kernel that started an iteration (mde_solver_debug_times)
  LsState ls;
  LbfgsState lb;
};

__device__ __forceinline__ bool off(const int* flag) { return *flag == 0; }

// Fixed-order reduction of K sums over nb block partials into smem out[K]; all threads of the block call.
// Stage 1: thread t owns (k = t % K, segment = t / K) and walks blocks segment, segment + S, ... in batches of
// 16 independent coalesced loads (through L2: the partials may come from other SMs of the same launch).
// Stage 2: one warp per output combines the S segment sums with a fixed shuffle tree.  The summation order
// depends only on (nb, K, blockDim), so scalars are bit-reproducible for a given launch shape.
template <bool MAXLAST>
__device__ void reduce_partials(const double* __restrict__ part, int nb, int K, double* out) {
  __shared__ double red_buf[256];
  const int T = blockDim.x < 256 ? blockDim.x : 256;
  const int S = T / K;  // segments (K <= 44 < T)
  const int k = threadIdx.x % K, seg = threadIdx.x / K;
  const bool is_max = MAXLAST && (k == K - 1);
  if (threadIdx.x < S * K) {
    constexpr int U = 16;
    double s = 0.0;
    for (int b0 = seg; b0 < nb; b0 += U * S) {
      double v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int b = b0 + u * S;
        v[u] = (b < nb) ? __ldcg(part + (int64_t)b * K + k) : 0.0;  // 0 is neutral for the sums and for max |.|
      }
#pragma unroll
      for (int u = 0; u < U; ++u) s = is_max ? fmax(s, v[u]) : s + v[u];
    }
    red_buf[seg * K + k] = s;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (int)(blockDim.x >> 5);
  for (int kk = w; kk < K; kk += nw) {  // warp-uniform trip count
    const bool mx = MAXLAST && (kk == K - 1);
    double s = 0.0;
    for (int q = lane; q < S; q += 32) { const double v = red_buf[q * K + kk]; s = mx ? fmax(s, v) : s + v; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double v = __shfl_xor_sync(kFull, s, o); s = mx ? fmax(s, v) : s + v; }
    if (lane == 0) out[kk] = s;
  }
  __syncthreads();
}

// "Last block done": every block publishes its partials, takes a ticket, and the block that draws the
// last ticket runs the scalar epilogue in the same launch (saves one dependent launch per reduction).
// The epilogue reads the partials in a fixed order, so the result does not depend on which block is last.
__device__ bool last_block_done(unsigned int* counter) {
  __shared__ int s_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned total = gridDim.x * gridDim.y;
    const unsigned t = atomicAdd(counter, 1u);
    s_last = (t == total - 1u) ? 1 : 0;
    if (s_last) *counter = 0u;
  }
  __syncthreads();
  if (s_last) __threadfence();
  return s_last != 0;
}

struct Tail {              // what a fused scalar epilogue needs
  int fuse;                // 0: separate scalar kernel follows; 1: run the epilogue in the last block
  int mode;                // grad_dots: 1 = line-search update, 2 = fresh evaluation
  const double* lpart;     // loss partials of the distortion launch
  int nl;
  const float* tail;       // (hi, lo) of the all-reduced loss (multi-GPU)
  double p_total;
  int64_t n_rows;
  double inv_n;            // 1 / n_rows
  cudaGraphConditionalHandle h_while;
};

__device__ void direction_scalar_body(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks,
                                      unsigned char* smem);
__device__ void ls_init_body(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks,
                             int64_t n_rows, cudaGraphConditionalHandle h_while);
__device__ void ls_update_body(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                               const float* __restrict__ tail, const double* __restrict__ dpart, int nd,
                               double p_total, cudaGraphConditionalHandle h_while);
__device__ void fresh_finish_body(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                                  const float* __restrict__ tail, const double* __restrict__ dpart, int nd,
                                  double p_total);
__device__ void iter_end_body(SolverState* __restrict__ S, cudaGraphConditionalHandle h_if_next);
__device__ void step_end_body(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                              const float* __restrict__ tail, const double* __restrict__ dpart, int nd,
                              double p_total);

constexpr int kScalarSmemBytes = (int)(sizeof(double) * (kMaxSlices * kDotsPerSlice + 5 * kSlots) + 64 + sizeof(LbfgsState));

// ---------------------------------------------------------------------------------------
// P1: candidate pair + all dot products of the history against (y_c, s_c, g)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kVecThreads, 2)
lbfgs_dots_kernel(SolverState* __restrict__ S, const float* __restrict__ g, const float* __restrict__ gprev,
                  const float* __restrict__ d, float* __restrict__ Sb, float* __restrict__ Yb,
                  int64_t npad, double* __restrict__ part, Tail tl, const int* __restrict__ gate) {
  if (off(&S->active)) return;
  if (gate != nullptr && off(gate)) return;
  // reduction tile: 27 rows x 256 threads of fp32 partials (used twice: 54 sums), later the scalar epilogue's scratch
  constexpr int kHalf = kDotsPerSlice / 2;
  __shared__ __align__(16) unsigned char raw[sizeof(float) * kHalf * kVecThreads];
  static_assert(sizeof(raw) >= kScalarSmemBytes, "scalar epilogue must fit in the reduction tile");
  __shared__ const float* sp[kPairsPerSlice];
  __shared__ const float* yp[kPairsPerSlice];
  const int slice = blockIdx.y;
  const int count = S->lb.count;
  const bool skip = (S->lb.n_iter == 0) || (slice > 0 && slice * kPairsPerSlice >= count);
  if (!skip) {
  const float t = (float)S->t_last;
  float* sc = Sb + (int64_t)S->lb.cand * npad;
  float* yc = Yb + (int64_t)S->lb.cand * npad;
  if (threadIdx.x < kPairsPerSlice) {
    const int lj = slice * kPairsPerSlice + threadIdx.x;
    const int q = (lj < count) ? S->lb.order[lj] : 0;
    sp[threadIdx.x] = Sb + (int64_t)q * npad;
    yp[threadIdx.x] = Yb + (int64_t)q * npad;
  }
  __syncthreads();
  int nval = count - slice * kPairsPerSlice;  // pairs of this slice (block-uniform)
  if (nval > kPairsPerSlice) nval = kPairsPerSlice;
  // fp32 per-thread partial sums (at the bench size a thread owns ONE float4; at 1e7 rows ~130): the block and
  // grid stages below run in fp64.  The reference accumulates the same dot products in fp32 end to end.
  float acc[kDotsPerSlice];
#pragma unroll
  for (int k = 0; k < kDotsPerSlice; ++k) acc[k] = 0.0f;
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 G = reinterpret_cast<const float4*>(g)[i];
    const float4 P = reinterpret_cast<const float4*>(gprev)[i];
    const float4 D = reinterpret_cast<const float4*>(d)[i];
    const float gv[4] = {G.x, G.y, G.z, G.w};
    const float yv[4] = {G.x - P.x, G.y - P.y, G.z - P.z, G.w - P.w};
    const float sv[4] = {D.x * t, D.y * t, D.z * t, D.w * t};
    if (slice == 0) {
      reinterpret_cast<float4*>(yc)[i] = make_float4(yv[0], yv[1], yv[2], yv[3]);
      reinterpret_cast<float4*>(sc)[i] = make_float4(sv[0], sv[1], sv[2], sv[3]);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        acc[0] += yv[q] * sv[q]; acc[1] += yv[q] * yv[q];
        acc[2] += sv[q] * gv[q]; acc[3] += yv[q] * gv[q];
      }
    }
#pragma unroll
    for (int j = 0; j < kPairsPerSlice; ++j) {
      if (j < nval) {
        const float4 A = reinterpret_cast<const float4*>(sp[j])[i];
        const float4 B = reinterpret_cast<const float4*>(yp[j])[i];
        const float av[4] = {A.x, A.y, A.z, A.w};
        const float bv[4] = {B.x, B.y, B.z, B.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          acc[4 + 5 * j + 0] += av[q] * yv[q];
          acc[4 + 5 * j + 1] += bv[q] * yv[q];
          acc[4 + 5 * j + 2] += sv[q] * bv[q];
          acc[4 + 5 * j + 3] += av[q] * gv[q];
          acc[4 + 5 * j + 4] += bv[q] * gv[q];
        }
      }
    }
  }
  // block reduction through a transposed shared-memory tile, two halves of 27 sums: each warp sums whole rows in
  // fp64 (8 conflict-free loads per lane + one shuffle tree per row)
  float (*tile)[kVecThreads] = reinterpret_cast<float (*)[kVecThreads]>(raw);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double* o = part + ((int64_t)slice * gridDim.x + blockIdx.x) * kDotsPerSlice;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (h) __syncthreads();
#pragma unroll
    for (int k = 0; k < kHalf; ++k) tile[k][threadIdx.x] = acc[h * kHalf + k];
    __syncthreads();
    for (int k = w; k < kHalf; k += kVecThreads / 32) {
      double sum = 0.0;
#pragma unroll
      for (int q = 0; q < kVecThreads / 32; ++q) sum += (double)tile[k][lane + 32 * q];
      sum = warp_sum(sum);
      if (lane == 0) o[h * kHalf + k] = sum;
    }
  }
  }  // !skip
  if (tl.fuse && last_block_done(&S->tickets[0])) direction_scalar_body(S, part, gridDim.x, raw);
}

// ---------------------------------------------------------------------------------------
// S1: statistics of the iteration start + history update + two-loop in Gram form
// ---------------------------------------------------------------------------------------
// Block-cooperative version of mde_logic.h::lbfgs_direction (same decisions, same formulas): thread 0
// takes the accept / evict decision, all threads move the Gram matrices, warp 0 runs the two-loop
// recursion with lane j owning al_j and c_j (each step is one masked warp reduction instead of a
// serial inner loop).  `dots` = [sj_yc | yj_yc | sc_yj | sj_g | yj_g], each kSlots long, in shared memory.
__device__ void lbfgs_direction_block(LbfgsState& B, double* dots, double ys, double yy, double sc_g, double yc_g,
                                      int* flags /* smem: [0]=first [1]=accepted [2]=evicted [3]=h before append */) {
  double* sj_yc = dots; double* yj_yc = dots + kSlots; double* sc_yj = dots + 2 * kSlots;
  double* sj_g = dots + 3 * kSlots; double* yj_g = dots + 4 * kSlots;
  const int tid = threadIdx.x;
  if (tid == 0) {
    B.n_iter += 1;
    flags[0] = (B.n_iter == 1);
    flags[1] = flags[2] = 0;
    if (flags[0]) { B.count = 0; B.H_diag = 1.0; B.cg = -1.0; }
    else if ((float)ys > 1e-10f) {
      flags[1] = 1;
      int h = B.count;
      const int c = B.cand;
      if (h == B.memory) {
        flags[2] = 1;
        const int freed = B.order[0];
        for (int j = 1; j < h; ++j) B.order[j - 1] = B.order[j];
        h -= 1;
        B.order[h] = c; B.cand = freed;
      } else {
        B.order[h] = c;
        unsigned long long used = 0ull;
        for (int j = 0; j <= h; ++j) used |= 1ull << B.order[j];
        int f = 0;
        while (f < kSlots - 1 && ((used >> f) & 1ull)) ++f;
        B.cand = f;
      }
      flags[3] = h;
      B.count = h + 1;
      B.H_diag = (double)((float)ys / (float)yy);
    }
  }
  __syncthreads();
  if (flags[0]) return;
  if (flags[2]) {  // evict the oldest pair: shift matrices and dot arrays up-left by one
    const int h_old = flags[3] + 1;
    double a[4], b[4];
    int n = 0;
    for (int k = tid; k < (h_old - 1) * (h_old - 1); k += blockDim.x) {
      int i = k / (h_old - 1) + 1, j = k % (h_old - 1) + 1;
      a[n] = B.SY[i][j]; b[n] = B.YY[i][j]; ++n;
    }
    double v[5] = {0, 0, 0, 0, 0};
    if (tid >= 1 && tid < h_old) { v[0] = sj_yc[tid]; v[1] = yj_yc[tid]; v[2] = sc_yj[tid]; v[3] = sj_g[tid]; v[4] = yj_g[tid]; }
    __syncthreads();
    n = 0;
    for (int k = tid; k < (h_old - 1) * (h_old - 1); k += blockDim.x) {
      int i = k / (h_old - 1), j = k % (h_old - 1);
      B.SY[i][j] = a[n]; B.YY[i][j] = b[n]; ++n;
    }
    if (tid >= 1 && tid < h_old) { sj_yc[tid - 1] = v[0]; yj_yc[tid - 1] = v[1]; sc_yj[tid - 1] = v[2]; sj_g[tid - 1] = v[3]; yj_g[tid - 1] = v[4]; }
    __syncthreads();
  }
  if (flags[1]) {  // append the candidate as the newest pair
    const int h = flags[3];
    if (tid < h) {
      B.SY[tid][h] = sj_yc[tid]; B.SY[h][tid] = sc_yj[tid];
      B.YY[tid][h] = yj_yc[tid]; B.YY[h][tid] = yj_yc[tid];
    }
    if (tid == 0) { B.SY[h][h] = ys; B.YY[h][h] = yy; sj_g[h] = sc_g; yj_g[h] = yc_g; }
    __syncthreads();
  }
  if (tid < 32) {
    // Two-loop recursion (lbfgs.py:488-507) on the Gram matrices, written as two triangular
    // substitutions in column-oriented form: lane k owns its own right-hand side, each step is one
    // divide + one broadcast + one FMA (no per-step warp reduction).
    //   loop 1 (newest -> oldest):  R al = -S^T g     with R = upper triangle of SY (s_i . y_j, j >= i)
    //   loop 2 (oldest -> newest):  c_i = al_i - (H (Y^T q)_i + sum_{j<i} c_j SY[j][i]) / SY[i][i]
    const int lane = tid, h = B.count;
    const double H = B.H_diag;
    // fp64 division is a ~300-cycle software routine: take the h reciprocals of the pivots in parallel (one per
    // lane) so that the two dependent chains below are shuffle + multiply + FMA only
    const double inv_piv = (lane < h) ? 1.0 / B.SY[lane][lane] : 0.0;
    double rhs = (lane < h) ? -sj_g[lane] : 0.0;
    double al = 0.0;
    for (int i = h - 1; i >= 0; --i) {
      const double ali = __shfl_sync(kFull, rhs, i) * __shfl_sync(kFull, inv_piv, i);
      if (lane == i) al = ali;
      if (lane < i) rhs -= ali * B.SY[lane][i];
    }
    // (Y^T q)_i = -y_i.g - sum_j al_j y_i.y_j : every lane needs all al_j
    double yq = (lane < h) ? -yj_g[lane] : 0.0;
    for (int j = 0; j < h; ++j) {
      const double alj = __shfl_sync(kFull, al, j);
      if (lane < h) yq -= alj * B.YY[lane][j];
    }
    double acc = H * yq, cc = 0.0;
    for (int j = 0; j < h; ++j) {
      const double accj = __shfl_sync(kFull, acc, j);
      const double alj = __shfl_sync(kFull, al, j);
      const double ccj = alj - accj * __shfl_sync(kFull, inv_piv, j);
      if (lane == j) cc = ccj;
      if (lane > j && lane < h) acc += ccj * B.SY[j][lane];
    }
    if (lane < h) { B.cs[lane] = cc; B.cy[lane] = -H * al; }
    if (lane == 0) B.cg = -H;
  }
}

__device__ void direction_scalar_body(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks,
                                      unsigned char* smem) {
  // carve: history state (Gram matrices included) | block sums | per-pair dots | flags
  LbfgsState& sB = *reinterpret_cast<LbfgsState*>(smem);
  double* sums = reinterpret_cast<double*>(smem + sizeof(LbfgsState));
  double* dots = sums + kMaxSlices * kDotsPerSlice;
  int* flags = reinterpret_cast<int*>(dots + 5 * kSlots);
  static_assert(sizeof(LbfgsState) % sizeof(double) == 0, "LbfgsState must be a whole number of doubles");
  static_assert(kMaxMemory <= 32, "the two-loop recursion maps one pair per lane");
  // The history state is staged through registers so that its loads are in flight together with the loads of
  // the reductions below (both come from L2; issuing them back to back hides one round trip).
  constexpr int kStateDoubles = (int)(sizeof(LbfgsState) / sizeof(double));
  constexpr int kStatePerThread = (kStateDoubles + 255) / 256;
  const int count = S->lb.count;
  const int n_iter = S->lb.n_iter;
  double stage[kStatePerThread];
  {
    const double* src = reinterpret_cast<const double*>(&S->lb);
#pragma unroll
    for (int q = 0; q < kStatePerThread; ++q) {
      const int k = (int)threadIdx.x + q * 256;
      stage[q] = (threadIdx.x < 256 && k < kStateDoubles) ? __ldcg(src + k) : 0.0;
    }
  }
  int slices = (count + kPairsPerSlice - 1) / kPairsPerSlice;
  if (slices < 1) slices = 1;
  if (n_iter > 0) {
    for (int s = 0; s < slices; ++s)
      reduce_partials<false>(part + (int64_t)s * nblocks * kDotsPerSlice, nblocks, kDotsPerSlice,
                             sums + s * kDotsPerSlice);
  }
  {
    double* dst = reinterpret_cast<double*>(&sB);
#pragma unroll
    for (int q = 0; q < kStatePerThread; ++q) {
      const int k = (int)threadIdx.x + q * 256;
      if (threadIdx.x < 256 && k < kStateDoubles) dst[k] = stage[q];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    // callback of LBFGS.step (optim.py:94-96): loss and ||X.grad||_F at the iteration start
    const int it = S->iter;
    const double resid = (double)sqrtf((float)S->gg);
    if (it < S->max_stats) { S->avg[it] = S->loss; S->resid[it] = resid; }
    S->stop_after = (resid <= S->eps) ? 1 : 0;
  }
  if (threadIdx.x < count) {
    const int j = threadIdx.x;
    const double* b = sums + (j / kPairsPerSlice) * kDotsPerSlice + 4 + 5 * (j % kPairsPerSlice);
    dots[j] = b[0]; dots[kSlots + j] = b[1]; dots[2 * kSlots + j] = b[2]; dots[3 * kSlots + j] = b[3];
    dots[4 * kSlots + j] = b[4];
  }
  __syncthreads();
  if (n_iter > 0) lbfgs_direction_block(sB, dots, sums[0], sums[1], sums[2], sums[3], flags);
  else lbfgs_direction_block(sB, dots, 0.0, 0.0, 0.0, 0.0, flags);
  __syncthreads();
  {
    double* dst = reinterpret_cast<double*>(&S->lb);
    const double* src = reinterpret_cast<const double*>(&sB);
    for (int k = threadIdx.x; k < (int)(sizeof(LbfgsState) / sizeof(double)); k += blockDim.x) dst[k] = src[k];
  }
}

__global__ void __launch_bounds__(256)
direction_scalar_kernel(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks) {
  if (off(&S->active)) return;
  __shared__ __align__(16) unsigned char raw[kScalarSmemBytes];
  direction_scalar_body(S, part, nblocks, raw);
}

// ---------------------------------------------------------------------------------------
// P2: d = cg*g + sum_j cs_j S_j + cy_j Y_j ; g_prev = g ; x_init = X ; partial g.d, d.d, X.X, max|d|
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kVecThreads)
direction_apply_kernel(SolverState* __restrict__ S, const float* __restrict__ g, float* __restrict__ gprev,
                       float* __restrict__ d, const float* __restrict__ X, float* __restrict__ xinit,
                       const float* __restrict__ Sb, const float* __restrict__ Yb, int64_t npad,
                       double* __restrict__ part, int mcols, Tail tl, const int* __restrict__ gate) {
  if (off(&S->active)) return;
  if (gate != nullptr && off(gate)) return;
  __shared__ float cs[kMaxMemory], cy[kMaxMemory];
  __shared__ const float* ps[kMaxMemory];
  __shared__ const float* py[kMaxMemory];
  const int count = S->lb.count;
  const float cg = (float)S->lb.cg;
  if (threadIdx.x < count) {
    cs[threadIdx.x] = (float)S->lb.cs[threadIdx.x];
    cy[threadIdx.x] = (float)S->lb.cy[threadIdx.x];
    int q = S->lb.order[threadIdx.x];
    ps[threadIdx.x] = Sb + (int64_t)q * npad;
    py[threadIdx.x] = Yb + (int64_t)q * npad;
  }
  __syncthreads();
  constexpr int KA = 11;  // g.d, d.d, X.X, column sums of X (4) and of d (4)
  double acc[KA];
  float fa[KA];
#pragma unroll
  for (int k = 0; k < KA; ++k) { acc[k] = 0.0; fa[k] = 0.0f; }
  float mx = 0.0f;
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int cnt = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 Xv = reinterpret_cast<const float4*>(X)[i];
    float r[4] = {cg * G.x, cg * G.y, cg * G.z, cg * G.w};
    for (int j = 0; j < count; ++j) {
      float4 A = reinterpret_cast<const float4*>(ps[j])[i];
      float4 B = reinterpret_cast<const float4*>(py[j])[i];
      r[0] += cs[j] * A.x + cy[j] * B.x; r[1] += cs[j] * A.y + cy[j] * B.y;
      r[2] += cs[j] * A.z + cy[j] * B.z; r[3] += cs[j] * A.w + cy[j] * B.w;
    }
    reinterpret_cast<float4*>(d)[i] = make_float4(r[0], r[1], r[2], r[3]);
    reinterpret_cast<float4*>(gprev)[i] = G;
    reinterpret_cast<float4*>(xinit)[i] = Xv;
    fa[0] += G.x * r[0] + G.y * r[1] + G.z * r[2] + G.w * r[3];
    fa[1] += r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
    fa[2] += Xv.x * Xv.x + Xv.y * Xv.y + Xv.z * Xv.z + Xv.w * Xv.w;
    mx = fmaxf(mx, fmaxf(fmaxf(fabsf(r[0]), fabsf(r[1])), fmaxf(fabsf(r[2]), fabsf(r[3]))));
    // column sums (rows are m floats; 4 % m == 0 so element q of a float4 belongs to column q % m)
    if (mcols == 1) {
      fa[3] += Xv.x + Xv.y + Xv.z + Xv.w; fa[7] += r[0] + r[1] + r[2] + r[3];
    } else if (mcols == 2) {
      fa[3] += Xv.x + Xv.z; fa[4] += Xv.y + Xv.w; fa[7] += r[0] + r[2]; fa[8] += r[1] + r[3];
    } else if (mcols == 4) {
      fa[3] += Xv.x; fa[4] += Xv.y; fa[5] += Xv.z; fa[6] += Xv.w;
      fa[7] += r[0]; fa[8] += r[1]; fa[9] += r[2]; fa[10] += r[3];
    }
    if (++cnt == 16) {
#pragma unroll
      for (int k = 0; k < KA; ++k) { acc[k] += (double)fa[k]; fa[k] = 0.0f; }
      cnt = 0;
    }
  }
#pragma unroll
  for (int k = 0; k < KA; ++k) acc[k] += (double)fa[k];
  __shared__ double sm[KA * 32];
  __shared__ float smx[32];
  block_sum<KA>(acc, sm);
  mx = warp_max(mx);
  if ((threadIdx.x & 31) == 0) smx[threadIdx.x >> 5] = mx;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m2 = 0.0f;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m2 = fmaxf(m2, smx[w]);
    double* o = part + (int64_t)blockIdx.x * (KA + 1);
#pragma unroll
    for (int k = 0; k < KA; ++k) o[k] = acc[k];
    o[KA] = (double)m2;
  }
  if (tl.fuse && last_block_done(&S->tickets[1])) ls_init_body(S, part, gridDim.x, tl.n_rows, tl.h_while);
}

// S2: finalize g.d, |d|, |X|; initial step; arm the line search (lbfgs.py:521-549)
__device__ void ls_init_body(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks,
                             int64_t n_rows, cudaGraphConditionalHandle h_while) {
  __shared__ double out[12];
  reduce_partials<true>(part, nblocks, 12, out);
  if (threadIdx.x == 0) {
    S->gtd = (float)out[0]; S->dd = out[1]; S->xx = out[2]; S->dmax = (float)out[11];
    const double inv_n = 1.0 / (double)n_rows;
#pragma unroll
    for (int c = 0; c < 4; ++c) { S->mu_x[c] = (float)(out[3 + c] * inv_n); S->mu_d[c] = (float)(out[7 + c] * inv_n); }
    double t0 = 1.0;
    if (S->lb.n_iter == 1) {  // t = min(1, 1/||g||_1) * lr
      float inv = 1.0f / (float)S->g1;
      t0 = (inv < 1.0f) ? (double)inv : 1.0;
    }
    LsState L;
    ls_begin(L, t0, S->loss, (float)out[0], (float)out[11]);
    S->ls = L;
    S->ls_active = 1;
    if (h_while) cudaGraphSetConditional(h_while, 1u);  // enter the device-side trial loop
  }
}

__global__ void __launch_bounds__(256)
ls_init_kernel(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks, int64_t n_rows,
               cudaGraphConditionalHandle h_while) {
  if (off(&S->active)) return;
  ls_init_body(S, part, nblocks, n_rows, h_while);
}

// graph mode: gate of the IF node around the fresh evaluation
__global__ void fresh_gate_kernel(const SolverState* __restrict__ S, cudaGraphConditionalHandle h_if) {
  if (threadIdx.x == 0) cudaGraphSetConditional(h_if, (S->active && S->need_fresh) ? 1u : 0u);
}

// ---------------------------------------------------------------------------------------
// trial point: X = x_init + t*d  (LBFGS._add_grad, lbfgs.py:350-357); FINAL uses t_accept
// ---------------------------------------------------------------------------------------
// center_m = 0: plain axpy.  center_m in {1,2,4}: the Centered projection (constraints.py:106-111) is
// folded in analytically, mean(x_init + t d) = mean(x_init) + t mean(d) with both means taken in the
// direction pass, so a trial point costs one pass and no reduction.  `gz` (trial only): gradient buffer
// zeroed in the same pass for the scatter kernel that follows.
template <bool FINAL>
__global__ void __launch_bounds__(kVecThreads)
trial_axpy_kernel(SolverState* __restrict__ S, const float* __restrict__ xinit, const float* __restrict__ d,
                  float* __restrict__ X, int64_t npad, int64_t nvalid, int center_m, float* __restrict__ gz,
                  int fuse_end, cudaGraphConditionalHandle h_if_next) {
  if (off(&S->active)) return;
  if (!FINAL && off(&S->ls_active)) return;
  const float t = FINAL ? (float)S->ls.t_accept : (float)S->ls.t;
  // FINAL: the accepted step is usually the last trial evaluated -- X already holds exactly
  // project(x_init + t d) (same kernel, same inputs, deterministic), so only the epilogue is needed.
  const bool same_point = FINAL && center_m != 0 && (S->ls.t_accept == S->t_eval);
  float mu[4] = {0.f, 0.f, 0.f, 0.f};
  if (center_m == 1) { float v = S->mu_x[0] + t * S->mu_d[0]; mu[0] = mu[1] = mu[2] = mu[3] = v; }
  else if (center_m == 2) {
    float v0 = S->mu_x[0] + t * S->mu_d[0], v1 = S->mu_x[1] + t * S->mu_d[1];
    mu[0] = mu[2] = v0; mu[1] = mu[3] = v1;
  } else if (center_m == 4) {
#pragma unroll
    for (int c = 0; c < 4; ++c) mu[c] = S->mu_x[c] + t * S->mu_d[c];
  }
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4 + 1 && !same_point; i += stride) {
    if (i < n4) {
      float4 A = reinterpret_cast<const float4*>(xinit)[i];
      float4 D = reinterpret_cast<const float4*>(d)[i];
      float4 R = make_float4(fmaf(t, D.x, A.x) - mu[0], fmaf(t, D.y, A.y) - mu[1], fmaf(t, D.z, A.z) - mu[2],
                             fmaf(t, D.w, A.w) - mu[3]);
      if (center_m != 0 && 4 * i + 3 >= nvalid) {  // keep the zero padding behind the last row
        if (4 * i + 0 >= nvalid) R.x = 0.f;
        if (4 * i + 1 >= nvalid) R.y = 0.f;
        if (4 * i + 2 >= nvalid) R.z = 0.f;
        if (4 * i + 3 >= nvalid) R.w = 0.f;
      }
      reinterpret_cast<float4*>(X)[i] = R;
    }
    if (!FINAL && gz != nullptr) reinterpret_cast<float4*>(gz)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (FINAL && fuse_end && last_block_done(&S->tickets[3])) iter_end_body(S, h_if_next);
}

__global__ void __launch_bounds__(kVecThreads)
zero_kernel(const int* flag, float* __restrict__ p, int64_t n4) {
  if (off(flag)) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride)
    reinterpret_cast<float4*>(p)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
}

// anchored constraint (pymde/constraints.py:114-164): overwrite / zero anchor rows
__global__ void anchor_rows_kernel(const int* flag, float* __restrict__ Z, const int64_t* __restrict__ anchors,
                                   const float* __restrict__ values, int64_t na, int m) {
  if (off(flag)) return;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= na * m) return;
  int64_t a = anchors[i / m];
  Z[a * m + (i % m)] = values ? values[i] : 0.0f;
}

// mode 2, multi-GPU: the all-reduced [gradient | loss] becomes the solver's gradient buffer -- only when the
// step really evaluated (the all-reduce itself cannot be gated, so it works on a staging buffer)
__global__ void __launch_bounds__(kVecThreads)
gated_copy_kernel(const int* flag, const float* __restrict__ src, float* __restrict__ dst, int64_t n4) {
  if (off(flag)) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride)
    reinterpret_cast<float4*>(dst)[i] = reinterpret_cast<const float4*>(src)[i];
}

// multi-GPU: pack this rank's loss sum behind the gradient as (hi, lo) floats
__global__ void __launch_bounds__(256)
pack_loss_kernel(const int* flag, const double* __restrict__ lpart, int nl, float* __restrict__ tail) {
  if (off(flag)) return;
  __shared__ double out[1];
  reduce_partials<false>(lpart, nl, 1, out);
  if (threadIdx.x == 0) {
    float hi = (float)out[0];
    tail[0] = hi;
    tail[1] = (float)(out[0] - (double)hi);
  }
}

// ---------------------------------------------------------------------------------------
// Multi-GPU (SURVEY section 8e): edge shards, X replicated, ONE all-reduce of [gradient | loss] per evaluation.
// The all-reduce is done by OUR kernels over NVLink peer memory (cudaIpc-mapped buffers of the other ranks), not by
// a host-side NCCL call: plain kernel nodes, so the sharded solve runs the same CUDA graph of gated steps as one
// GPU, and a gated-off step costs nothing.  Every rank sums the peers' partial buffers in RANK ORDER, so all ranks
// hold bit-identical gradients (the replicated Wolfe / L-BFGS decisions depend on it).
//   small buffers (<= kOneShotBytes): one-shot -- every rank reads all W partial buffers and writes g;
//   large buffers: two-shot -- rank r reduces chunk r in place (reduce-scatter), then everybody gathers the
//   W reduced chunks (all-gather): 2 (W-1)/W of the buffer over NVLink instead of (W-1).
// Handshake: monotonically increasing epochs in per-rank flag arrays (st.release.sys / ld.acquire.sys),
// fa = "my partial buffer is complete", fb = "my chunk is reduced", fd = "I have finished reading the peers".
// Spins are bounded: a peer that never arrives sets the solver's error word instead of hanging the GPU.
// ---------------------------------------------------------------------------------------
constexpr int kMaxWorld = 8;
constexpr int kCommThreads = 512;
constexpr int64_t kOneShotBytes = 4ll << 20;
constexpr long long kSpinLimitCycles = 20000000000ll;  // ~10 s at 2 GHz

struct Comm {
  int rank, world;
  float* buf[kMaxWorld];      // partial [gradient | hi lo] buffer of every rank (peer-mapped)
  unsigned* fa[kMaxWorld];    // flag arrays of every rank: f?[q][r] is written by rank r, polled by rank q
  unsigned* fb[kMaxWorld];
  unsigned* fd[kMaxWorld];
  unsigned* epoch;            // local: all-reduces completed so far
  unsigned int* ticket;       // local last-block-done counter
  // push path (large buffers): peers WRITE into these parts of a rank's region
  float* gout[kMaxWorld];     // the solver's gradient buffer g of every rank (npad + tail)
  float* recv[kMaxWorld];     // receive slots of every rank: recv[q] + r * slot_floats = rank r's copy of chunk q
  float* tails[kMaxWorld];    // (hi, lo) loss pair of rank r at tails[q] + 2 r
  int64_t slot_floats;        // floats per receive slot (>= chunk size)
};

__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Peer rows are read with plain (L1-allocating) 16-byte loads: a warp's 512 contiguous bytes travel as whole
// 128-byte lines over NVLink.  (ld.global.cg sustained only ~300 GB/s here: peer data is never cached in the local L2,
// so .cg requests go out sector by sector.)  Stale L1 lines cannot be hit: L1 is invalidated at every kernel launch
// and an address is read at most once per launch, after the acquire of its owner's flag.
__device__ __forceinline__ float4 ld_peer_f4(const float* p) { return *reinterpret_cast<const float4*>(p); }

// tell every rank "my epoch for this flag kind is `v`" (threads 0..W-1 of one block)
__device__ __forceinline__ void comm_signal(unsigned* const* flags, const Comm& c, unsigned v) {
  __threadfence_system();
  if ((int)threadIdx.x < c.world) st_release_sys(flags[threadIdx.x] + c.rank, v);
}
// wait until every rank has signalled epoch >= v in MY flag array; all threads of the block call
__device__ __forceinline__ void comm_wait(const unsigned* mine, const Comm& c, unsigned v, int* err) {
  if ((int)threadIdx.x < c.world) {
    const long long t0 = clock64();
    while ((int)(ld_acquire_sys(mine + threadIdx.x) - v) < 0) {
      if (clock64() - t0 > kSpinLimitCycles) { atomicExch(err, MDE_E_COMM); break; }
    }
  }
  __syncthreads();
}

// before this rank overwrites its partial buffer: every peer must have finished reading it
__device__ __forceinline__ void comm_wait_readers(const Comm& c, int* err) {
  comm_wait(c.fd[c.rank], c, *reinterpret_cast<volatile unsigned*>(c.epoch), err);
}

__device__ __forceinline__ void comm_wait_readers_fwd(const Comm* c, int* err) { comm_wait_readers(*c, err); }

// loss (hi, lo) pairs of all ranks summed in double, in rank order -> out[0..1]
__device__ __forceinline__ void comm_reduce_tail(const Comm& c, int64_t npad, float* out) {
  double sum = 0.0;
  for (int q = 0; q < c.world; ++q) {
    const volatile float* t = c.buf[q] + npad;
    sum += (double)t[0] + (double)t[1];
  }
  const float hi = (float)sum;
  out[0] = hi;
  out[1] = (float)(sum - (double)hi);
}

// One-shot: g[i] = sum_q buf_q[i] (rank order) for i < npad, tail summed in double.  MODE 0 = one-shot,
// 1 = reduce-scatter phase (chunk `rank` reduced in place), 2 = all-gather phase.
template <int PHASE>
__global__ void __launch_bounds__(kCommThreads)
allreduce_kernel(const int* __restrict__ flag, Comm c, float* __restrict__ g, int64_t npad, int* __restrict__ err) {
  if (off(flag)) return;
  const unsigned ep = *reinterpret_cast<volatile unsigned*>(c.epoch) + 1u;
  unsigned* const* sig = (PHASE == 2) ? c.fb : c.fa;
  if (blockIdx.x == 0) comm_signal(sig, c, ep);
  comm_wait(sig[c.rank], c, ep, err);
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr int U = 2;  // float4 per thread per trip; all U * world peer loads are issued before the first add
  if (PHASE == 0 || PHASE == 1) {
    // chunk q = [q * cs, min((q + 1) * cs, n4)) in float4 units; one-shot reduces everything, reduce-scatter its chunk
    const int64_t cs = (n4 + c.world - 1) / c.world;
    const int64_t lo = (PHASE == 0) ? 0 : (int64_t)c.rank * cs;
    const int64_t hi = (PHASE == 0) ? n4 : ((lo + cs < n4) ? lo + cs : n4);
    float* out = (PHASE == 0) ? g : c.buf[c.rank];
    for (int64_t i0 = lo + tid; i0 < hi; i0 += U * stride) {
      float4 v[kMaxWorld][U];
#pragma unroll
      for (int q = 0; q < kMaxWorld; ++q) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t i = i0 + u * stride;
          v[q][u] = (q < c.world && i < hi) ? ld_peer_f4(c.buf[q] + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float4 acc = v[0][u];
#pragma unroll
        for (int q = 1; q < kMaxWorld; ++q) {  // rank order: bit-identical sums on every rank (absent ranks add +0)
          if (q < c.world) { acc.x += v[q][u].x; acc.y += v[q][u].y; acc.z += v[q][u].z; acc.w += v[q][u].w; }
        }
        const int64_t i = i0 + u * stride;
        if (i < hi) reinterpret_cast<float4*>(out)[i] = acc;
      }
    }
    if (tid == 0) comm_reduce_tail(c, npad, g + npad);
  } else {
    const int64_t cs = (n4 + c.world - 1) / c.world;
    constexpr int UG = 8;
    for (int64_t i0 = tid; i0 < n4; i0 += UG * stride) {
      float4 v[UG];
#pragma unroll
      for (int u = 0; u < UG; ++u) {
        const int64_t i = i0 + u * stride;
        v[u] = (i < n4) ? ld_peer_f4(c.buf[(int)(i / cs)] + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
#pragma unroll
      for (int u = 0; u < UG; ++u) {
        const int64_t i = i0 + u * stride;
        if (i < n4) reinterpret_cast<float4*>(g)[i] = v[u];
      }
    }
  }
  if (PHASE != 1) {
    // the last block to finish tells the peers "I am done reading your buffers" and completes the epoch
    __shared__ int s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned t = atomicAdd(c.ticket, 1u);
      s_last = (t == gridDim.x - 1u) ? 1 : 0;
      if (s_last) *c.ticket = 0u;
    }
    __syncthreads();
    if (s_last) {
      comm_signal(c.fd, c, ep);
      if (threadIdx.x == 0) *c.epoch = ep;
    }
  }
}

// ---------------------------------------------------------------------------------------
// Large buffers: write-based ("push") all-reduce.  NVLink stores are posted, loads are round trips: the read-based
// reduce-scatter + all-gather above sustained ~300 GB/s per GPU on 80 MB gradients.  Here every byte crosses NVLink
// as a store:
//   K<0>  rank r copies chunk q of its partial buffer into rank q's receive slot r (all q != r) and its loss pair
//         into everybody's tails; last block: fence + flag fa
//   K<1>  wait fa of all ranks; rank q sums its W copies of chunk q IN RANK ORDER and stores the result into the
//         gradient buffer of EVERY rank (its own and the peers'); loss pairs summed in double; last block: fence + fb
//   K<2>  one block: wait fb of all ranks (every chunk of g has landed, every peer is done with my receive slots),
//         publish fd, complete the epoch
// ---------------------------------------------------------------------------------------
template <int STAGE>
__global__ void __launch_bounds__(kCommThreads)
allreduce_push_kernel(const int* __restrict__ flag, Comm c, int64_t npad, int* __restrict__ err) {
  if (off(flag)) return;
  const unsigned ep = *reinterpret_cast<volatile unsigned*>(c.epoch) + 1u;
  const int64_t n4 = npad >> 2;
  const int64_t cs = (n4 + c.world - 1) / c.world;  // chunk q = [q cs, min((q + 1) cs, n4)) in float4 units
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float* mine = c.buf[c.rank];
  if (STAGE == 2) {
    comm_wait(c.fb[c.rank], c, ep, err);
    comm_signal(c.fd, c, ep);
    if (threadIdx.x == 0) *c.epoch = ep;
    return;
  }
  if (STAGE == 0) {
    for (int dq = 1; dq < c.world; ++dq) {
      const int q = (c.rank + dq) % c.world;  // start with the next rank: the W ranks hit W different targets
      const int64_t lo = (int64_t)q * cs, hi = (lo + cs < n4) ? lo + cs : n4;
      float4* dst = reinterpret_cast<float4*>(c.recv[q] + (int64_t)c.rank * c.slot_floats);
      constexpr int U = 4;
      for (int64_t i0 = lo + tid; i0 < hi; i0 += U * stride) {
        float4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t i = i0 + u * stride;
          v[u] = (i < hi) ? reinterpret_cast<const float4*>(mine)[i] : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t i = i0 + u * stride;
          if (i < hi) dst[i - lo] = v[u];
        }
      }
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < c.world) {
      float* t = c.tails[threadIdx.x] + 2 * c.rank;
      t[0] = mine[npad];
      t[1] = mine[npad + 1];
    }
  } else {
    comm_wait(c.fa[c.rank], c, ep, err);
    const int64_t lo = (int64_t)c.rank * cs, hi = (lo + cs < n4) ? lo + cs : n4;
    constexpr int U = 2;
    for (int64_t i0 = lo + tid; i0 < hi; i0 += U * stride) {
      float4 v[kMaxWorld][U];
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r) {
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t i = i0 + u * stride;
          if (r < c.world && i < hi) {
            v[r][u] = (r == c.rank) ? reinterpret_cast<const float4*>(mine)[i]
                                    : __ldcg(reinterpret_cast<const float4*>(c.recv[c.rank] + (int64_t)r * c.slot_floats) + (i - lo));
          } else {
            v[r][u] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        float4 acc = v[0][u];
#pragma unroll
        for (int r = 1; r < kMaxWorld; ++r) {  // rank order: bit-identical on every rank (absent ranks add +0)
          if (r < c.world) { acc.x += v[r][u].x; acc.y += v[r][u].y; acc.z += v[r][u].z; acc.w += v[r][u].w; }
        }
        const int64_t i = i0 + u * stride;
        if (i < hi) {
          for (int dq = 0; dq < c.world; ++dq) {
            const int q = (c.rank + dq) % c.world;
            reinterpret_cast<float4*>(c.gout[q])[i] = acc;
          }
        }
      }
    }
    if (tid == 0) {  // every rank sums the same W pairs in the same order
      double sum = 0.0;
      for (int r = 0; r < c.world; ++r) {
        const volatile float* t = c.tails[c.rank] + 2 * r;
        sum += (double)t[0] + (double)t[1];
      }
      const float hi_f = (float)sum;
      c.gout[c.rank][npad] = hi_f;
      c.gout[c.rank][npad + 1] = (float)(sum - (double)hi_f);
    }
  }
  // the last block to finish publishes the stage: all stores of this launch are fenced before the flag
  __shared__ int s_last;
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(c.ticket, 1u);
    s_last = (t == gridDim.x - 1u) ? 1 : 0;
    if (s_last) *c.ticket = 0u;
  }
  __syncthreads();
  if (s_last) comm_signal(STAGE == 0 ? c.fa : c.fb, c, ep);
}

// T5: partial g.d, g.g, |g|_1
__global__ void __launch_bounds__(kVecThreads)
grad_dots_kernel(const int* flag, const float* __restrict__ g, const float* __restrict__ d, int64_t npad,
                 double* __restrict__ part, SolverState* __restrict__ S, Tail tl) {
  if (tl.mode == 3) {  // mode 2 step: `flag` is the evaluation gate; PH_MAT has no evaluation, only the epilogue
    if (off(&S->active)) return;
    if (S->g_mat) {  // the epilogue rewrites the gates: run it once every block has read them
      if (last_block_done(&S->tickets[2])) step_end_body(S, tl.lpart, tl.nl, tl.tail, part, gridDim.x, tl.p_total);
      return;
    }
  }
  if (off(flag)) return;
  double acc[3] = {0.0, 0.0, 0.0};
  float fa[3] = {0.0f, 0.0f, 0.0f};
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int cnt = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 D = reinterpret_cast<const float4*>(d)[i];
    fa[0] += G.x * D.x + G.y * D.y + G.z * D.z + G.w * D.w;
    fa[1] += G.x * G.x + G.y * G.y + G.z * G.z + G.w * G.w;
    fa[2] += fabsf(G.x) + fabsf(G.y) + fabsf(G.z) + fabsf(G.w);
    if (++cnt == 16) {
      for (int k = 0; k < 3; ++k) { acc[k] += (double)fa[k]; fa[k] = 0.0f; }
      cnt = 0;
    }
  }
  for (int k = 0; k < 3; ++k) acc[k] += (double)fa[k];
  __shared__ double sm[3 * 32];
  block_sum<3>(acc, sm);
  if (threadIdx.x == 0) {
    double* o = part + (int64_t)blockIdx.x * 3;
    o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
  }
  if (tl.fuse && last_block_done(&S->tickets[2])) {
    if (tl.mode == 1) ls_update_body(S, tl.lpart, tl.nl, tl.tail, part, gridDim.x, tl.p_total, tl.h_while);
    else if (tl.mode == 3) step_end_body(S, tl.lpart, tl.nl, tl.tail, part, gridDim.x, tl.p_total);
    else fresh_finish_body(S, tl.lpart, tl.nl, tl.tail, part, gridDim.x, tl.p_total);
  }
}

// loss of one evaluation as the reference sees it: fp32 mean, then float(...)
__device__ double eval_loss(const SolverState* S, const double* lpart, int nl, const float* tail, double* smem1,
                            double p_total) {
  double sum;
  if (S->world > 1) {
    sum = (double)tail[0] + (double)tail[1];
    __syncthreads();
  } else {
    reduce_partials<false>(lpart, nl, 1, smem1);
    sum = smem1[0];
  }
  return (double)(float)(sum / p_total);
}

// Both reductions an evaluation needs in ONE pass: loss partials of the scatter launch (nl x 1) and the
// (g.d, g.g, |g|_1) partials of the dots pass (nd x 3).  Same thread mapping and summation order as two
// reduce_partials calls (bit-identical results), but the loads of both are in flight together and there
// are two block barriers instead of four.  blockDim.x == 256.  out4 = [loss sum, g.d, g.g, |g|_1].
__device__ void reduce_loss_and_dots(const double* __restrict__ lpart, int nl, const double* __restrict__ dpart,
                                     int nd, double* out4) {
  __shared__ double buf_a[256], buf_b[256];
  constexpr int U = 4, SB = 85;  // 85 segments x 3 outputs = 255 threads for the dots
  const int t = threadIdx.x;
  const int kb = t % 3, segb = t / 3;
  const bool useb = t < 3 * SB;
  double a = 0.0, b = 0.0;
  for (int it = 0;; ++it) {
    const int ia0 = t + it * U * 256, ib0 = segb + it * U * SB;
    if (ia0 >= nl && (!useb || ib0 >= nd)) break;
    double va[U], vb[U];
#pragma unroll
    for (int u = 0; u < U; ++u) { const int i = ia0 + u * 256; va[u] = (i < nl) ? __ldcg(lpart + i) : 0.0; }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int i = ib0 + u * SB;
      vb[u] = (useb && i < nd) ? __ldcg(dpart + (int64_t)i * 3 + kb) : 0.0;
    }
#pragma unroll
    for (int u = 0; u < U; ++u) a += va[u];
#pragma unroll
    for (int u = 0; u < U; ++u) b += vb[u];
  }
  buf_a[t] = a;
  buf_b[t] = b;  // index seg * 3 + k == t for t < 255
  __syncthreads();
  const int lane = t & 31, w = t >> 5;
  if (w == 0) {
    double v = 0.0;
    for (int q = lane; q < 256; q += 32) v += buf_a[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    if (lane == 0) out4[0] = v;
  } else if (w <= 3) {
    const int k = w - 1;
    double v = 0.0;
    for (int q = lane; q < SB; q += 32) v += buf_b[q * 3 + k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
    if (lane == 0) out4[1 + k] = v;
  }
  __syncthreads();
}

// loss and (g.d, g.g, |g|_1) of one evaluation -> out3[0..2], returns the loss as the reference sees it
__device__ double eval_reductions(const SolverState* S, const double* lpart, int nl, const float* tail,
                                  const double* dpart, int nd, double p_total, double* out3) {
  __shared__ double r4[4];
  if (S->world > 1 || blockDim.x != 256) {
    __shared__ double l1[1];
    const double loss = eval_loss(S, lpart, nl, tail, l1, p_total);
    reduce_partials<false>(dpart, nd, 3, out3);
    return loss;
  }
  reduce_loss_and_dots(lpart, nl, dpart, nd, r4);
  if (threadIdx.x < 3) out3[threadIdx.x] = r4[1 + threadIdx.x];
  const double loss = (double)(float)(r4[0] / p_total);
  __syncthreads();
  return loss;
}

// S(fresh): closure() at the current iterate (lbfgs.py:426), no line search involved
__device__ void fresh_finish_body(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                                  const float* __restrict__ tail, const double* __restrict__ dpart, int nd,
                                  double p_total) {
  __shared__ double out[3];
  const double loss = eval_reductions(S, lpart, nl, tail, dpart, nd, p_total, out);
  if (threadIdx.x == 0) {
    S->loss = loss; S->gg = out[1]; S->g1 = out[2];
    S->func_evals += 1;
    S->pad0 = (int)S->func_evals;
  }
}

__global__ void __launch_bounds__(256)
fresh_finish_kernel(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                    const float* __restrict__ tail, const double* __restrict__ dpart, int nd, double p_total) {
  if (off(&S->active) || off(&S->need_fresh)) return;
  fresh_finish_body(S, lpart, nl, tail, dpart, nd, p_total);
}

// S(trial): feed (f_new, g.d) to the Wolfe state machine; decide the next step or finish
__device__ void ls_update_body(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                               const float* __restrict__ tail, const double* __restrict__ dpart, int nd,
                               double p_total, cudaGraphConditionalHandle h_while) {
  __shared__ double out[3];
  const double loss = eval_reductions(S, lpart, nl, tail, dpart, nd, p_total, out);
  if (threadIdx.x == 0) {
    S->gg = out[1]; S->g1 = out[2];
    S->func_evals += 1;
    S->pad0 = (int)S->func_evals;
    LsState L = S->ls;  // work on a register copy: the state machine touches ~30 fields
    S->t_eval = L.t;
    const bool finite = isfinite(out[1]);
    ls_on_result(L, loss, (float)out[0], finite);
    S->ls = L;
    if (L.phase == LS_DONE) {
      S->ls_active = 0;
      if (L.error) { S->error = MDE_E_NAN; S->active = 0; }
      S->t_last = L.t_accept;
      S->loss = (double)(float)L.f_accept;  // _cached_loss is an fp32 tensor (lbfgs.py:550)
    }
    if (h_while) cudaGraphSetConditional(h_while, (S->ls_active && S->active) ? 1u : 0u);
  }
}

__global__ void __launch_bounds__(256)
ls_update_kernel(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                 const float* __restrict__ tail, const double* __restrict__ dpart, int nd, double p_total,
                 cudaGraphConditionalHandle h_while) {
  if (off(&S->active) || off(&S->ls_active)) {
    if (h_while && threadIdx.x == 0) cudaGraphSetConditional(h_while, 0u);
    return;
  }
  ls_update_body(S, lpart, nl, tail, dpart, nd, p_total, h_while);
}

// S5: end of iteration (optim.py:135-173)
// `h_if_next`: in a graph that chains several iterations, the gate of the NEXT iteration's fresh-evaluation
// IF node is set here instead of by a separate one-thread kernel (0 = none).
__device__ void iter_end_body(SolverState* __restrict__ S, cudaGraphConditionalHandle h_if_next) {
  if (threadIdx.x != 0) return;
  const int it = S->iter;
  const double h = S->ls.t_accept;
  const double norm_x = (double)sqrtf((float)S->xx);
  const double pc = 100.0 * h * (double)sqrtf((float)S->dd) / norm_x;
  if (it < S->max_stats) { S->pct[it] = (double)(float)pc; S->steplen[it] = h; }
  S->iter = it + 1;
  if (S->stop_after) { S->converged = 1; S->active = 0; }
  else if (h == 0.0) { lbfgs_reset(S->lb, S->lb.memory); S->need_fresh = 1; }  // opt.reset()
  else S->need_fresh = 0;
  if (S->iter >= S->max_stats) S->active = 0;
  if (h_if_next) cudaGraphSetConditional(h_if_next, (S->active && S->need_fresh) ? 1u : 0u);
}

__global__ void iter_end_kernel(SolverState* __restrict__ S, cudaGraphConditionalHandle h_if_next) {
  if (off(&S->active)) return;  // the next IF handle keeps its default (0): nothing runs any more
  iter_end_body(S, h_if_next);
}

// ---------------------------------------------------------------------------------------
// mode 2: the solve as a flat chain of identical "steps" (no conditional graph nodes: an IF or WHILE node costs
// several times a dependent kernel node, tools/microbench/graph_overheads.cu measures them).  A step = direction kernels (gated) -> axpy -> retraction (gated)
// -> scatter kernel -> tangent projection -> dots + epilogue; it performs exactly one closure evaluation.
// The epilogue (last block of the dots kernel) advances a small phase machine and writes the gates the
// next step's kernels read:
//   PH_FRESH  closure at the current iterate (lbfgs n_iter == 0)           -> PH_DIR
//   PH_DIR    new direction + first line-search trial                      -> PH_TRIAL | PH_MAT | end of iteration
//   PH_TRIAL  another trial of the same line search                        -> PH_TRIAL | PH_MAT | end of iteration
//   PH_MAT    X = retract(x_init + t_accept d) when the accepted step is not the last one evaluated
//             (otherwise X already holds it bit for bit); no evaluation     -> end of iteration
// End of iteration (iter_end_body) -> PH_DIR, or PH_FRESH after a reset, or pause at iter_limit.
// ---------------------------------------------------------------------------------------
__device__ void set_phase(SolverState* __restrict__ S, int ph) {
  S->phase = ph;
  S->need_fresh = (ph == PH_FRESH) ? 1 : 0;
  const int on = S->active;
  S->g_dir = (on && ph == PH_DIR) ? 1 : 0;
  S->g_eval = (on && ph != PH_MAT) ? 1 : 0;
  S->g_mat = (on && ph == PH_MAT) ? 1 : 0;
  S->g_proj = (on && ph != PH_FRESH) ? 1 : 0;
}

__device__ void step_end_body(SolverState* __restrict__ S, const double* __restrict__ lpart, int nl,
                              const float* __restrict__ tail, const double* __restrict__ dpart, int nd,
                              double p_total) {
  const int ph = S->phase;  // uniform over the block
  if (ph == PH_FRESH) fresh_finish_body(S, lpart, nl, tail, dpart, nd, p_total);
  else if (ph != PH_MAT) ls_update_body(S, lpart, nl, tail, dpart, nd, p_total, 0);
  if (threadIdx.x != 0) return;
  if (S->error == MDE_E_COMM) S->active = 0;  // a peer never arrived: stop instead of timing out once per step
  int next = ph;
  bool end_of_iteration = false;
  if (ph == PH_FRESH) next = PH_DIR;
  else if (ph == PH_MAT) end_of_iteration = true;
  else if (S->ls_active) next = PH_TRIAL;
  else if (S->active) {  // line search finished (on SolverError `active` is already 0)
    if (S->ls.t_accept == S->t_eval) end_of_iteration = true;
    else next = PH_MAT;
  }
  if (end_of_iteration) {
    iter_end_body(S, 0);
    next = S->need_fresh ? PH_FRESH : PH_DIR;
    if (S->active && S->iter >= S->iter_limit) { S->active = 0; S->paused = 1; }
  }
  set_phase(S, next);
}

// ---------------------------------------------------------------------------------------
// mode 2, "late epilogue" steps (default; MDE_B200_LATE=0 keeps the chain above).  A step is
//     head -> vec -> [retraction kernels] -> scatter [-> all-reduce] [-> tangent projection]
// with ONE scalar stage, in the head kernel's last block:
//   head  reads g, g_prev, d, X and the history once: (g.d, g.g, |g|_1) of the evaluation the previous step left
//         pending, the history dots of the iteration that would start if that trial is accepted, column sums of g and
//         X (Centered).  Its blocks also fold the previous scatter launch's loss partials and the previous vec
//         kernel's (g.d, d.d, X.X, max|d|) partials into their rows, so the epilogue does one reduction.  Epilogue:
//         finish the previous step (line-search init if it was PH_DIR, Wolfe update, end of iteration), choose this
//         step's phase, and when an iteration starts: history update, two-loop, first step length, column means.
//   vec   PH_DIR: d = H g, g_prev = g, x_init = X and the first trial X = x_init + t0 d in ONE pass (t0 does not
//         depend on g.d: lbfgs.py:521-530); PH_TRIAL / PH_MAT: X = x_init + t d; every phase but PH_MAT: g = 0.
// 3 kernels and one one-block epilogue per evaluation instead of 5 and 3.  The history dots are SPECULATIVE (they
// assume the trial just evaluated, t = t_cur, is accepted, which the strong-Wolfe search does ~9 times out of 10);
// when it asks for another trial they are unused, when it accepts an earlier point (PH_MAT) the step after the
// materialisation recomputes them with the accepted t.
// ---------------------------------------------------------------------------------------
constexpr int kColG = kDotsPerSlice + 3;   // 57: column sums of g (4)
constexpr int kColX = kDotsPerSlice + 7;   // 61: column sums of X (4)
constexpr int kColLoss = kHeadAcc;         // 66: loss partial sum of the pending evaluation
constexpr int kColVec = kHeadAcc + 1;      // 67..70: g.d, d.d, X.X, max|d| of the pending PH_DIR step (max last)

__device__ void fill_head_desc(SolverState* S) {
  HeadDesc& h = S->hd;
  h.pend = S->pend; h.phase = S->phase; h.count = S->lb.count; h.n_iter = S->lb.n_iter; h.cand = S->lb.cand;
  h.t_cur = (float)S->t_cur; h.t_last = (float)S->t_last; h.pad = 0;
  for (int j = 0; j < 32; ++j) h.order[j] = (unsigned char)((j < kSlots) ? S->lb.order[j] : 0);
}

__device__ __forceinline__ unsigned long long gtime() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

__device__ void fresh_apply(SolverState* __restrict__ S, double loss, double gg, double g1) {
  S->loss = loss; S->gg = gg; S->g1 = g1;
  S->func_evals += 1;
  S->pad0 = (int)S->func_evals;
}

__device__ void ls_apply(SolverState* __restrict__ S, double loss, double gtd, double gg, double g1) {
  S->gg = gg; S->g1 = g1;
  S->func_evals += 1;
  S->pad0 = (int)S->func_evals;
  LsState L = S->ls;
  S->t_eval = L.t;
  ls_on_result(L, loss, (float)gtd, isfinite(gg));
  S->ls = L;
  if (L.phase == LS_DONE) {
    S->ls_active = 0;
    if (L.error) { S->error = MDE_E_NAN; S->active = 0; }
    S->t_last = L.t_accept;
    S->loss = (double)(float)L.f_accept;  // _cached_loss is an fp32 tensor (lbfgs.py:550)
  }
}

// The scalar stage of a late-epilogue step (last block of the head kernel).  The whole SolverState (history Gram
// matrices included, ~21 KB) is staged into shared memory with one cooperative copy, the phase machine, the
// line search and the two-loop recursion run on that copy, and it is written back once at the end: the serial
// part never waits for an L2 round trip.
constexpr int kStateDoubles = (int)(sizeof(SolverState) / sizeof(double));
constexpr int kLbOffsetDoubles = (int)(offsetof(SolverState, lb) / sizeof(double));
constexpr int kHeadSmemBytes = (int)(sizeof(SolverState) + sizeof(double) * (kMaxSlices * kHeadCols + 5 * kSlots) + 64);
static_assert(sizeof(SolverState) % sizeof(double) == 0 && offsetof(SolverState, lb) % sizeof(double) == 0, "staged as doubles");

// Fixed-order reduction of the head kernel's partial rows (kHeadCols doubles each, 16-byte aligned) into out[]:
// thread (segment, column pair) loads its rows as double2 -- all loads of a thread in flight together, one L2 round
// trip for <= 2 kNumSMs rows -- and adds them with two independent accumulators; then thread k combines the segments
// serially.  Dependent fp64 chains are what the one-block stage waits for (DADD + SHFL trees cost ~100 cycles a
// level with 8 resident warps), so there is no shuffle tree here.  Column `kmax` is a maximum, the others sums.
__device__ void reduce_head_rows(const double* __restrict__ part, int nb, double* __restrict__ out, int kmax) {
  constexpr int KP = kHeadCols / 2;            // column pairs
  constexpr int SEG = 256 / KP;                // segments
  constexpr int RB = 22;                       // rows per thread in flight (one batch covers 154 rows)
  __shared__ double red[SEG][kHeadCols];
  const int cp = threadIdx.x % KP, seg = threadIdx.x / KP;
  if (seg < SEG) {
    const bool mx = (2 * cp == kmax);
    double a0 = 0.0, a1 = 0.0, b0 = 0.0, b1 = 0.0;
    for (int base = seg; base < nb; base += RB * SEG) {
      double2 v[RB];
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        const int b = base + r * SEG;
        v[r] = (b < nb) ? __ldcg(reinterpret_cast<const double2*>(part + (int64_t)b * kHeadCols) + cp) : make_double2(0.0, 0.0);
      }
#pragma unroll
      for (int r = 0; r < RB; r += 2) {
        a0 = mx ? fmax(a0, v[r].x) : a0 + v[r].x; a1 = mx ? fmax(a1, v[r + 1].x) : a1 + v[r + 1].x;
        b0 += v[r].y; b1 += v[r + 1].y;
      }
    }
    red[seg][2 * cp] = mx ? fmax(a0, a1) : a0 + a1;
    red[seg][2 * cp + 1] = b0 + b1;
  }
  __syncthreads();
  if (threadIdx.x < kHeadCols) {
    const bool mx = ((int)threadIdx.x == kmax);
    double a0 = 0.0, a1 = 0.0;
#pragma unroll
    for (int q = 0; q + 1 < SEG; q += 2) {
      a0 = mx ? fmax(a0, red[q][threadIdx.x]) : a0 + red[q][threadIdx.x];
      a1 = mx ? fmax(a1, red[q + 1][threadIdx.x]) : a1 + red[q + 1][threadIdx.x];
    }
    if (SEG & 1) a0 = mx ? fmax(a0, red[SEG - 1][threadIdx.x]) : a0 + red[SEG - 1][threadIdx.x];
    out[threadIdx.x] = mx ? fmax(a0, a1) : a0 + a1;
  }
  __syncthreads();
}

__device__ void step_head_body(SolverState* __restrict__ S, const double* __restrict__ part, int nblocks, Tail tl,
                               unsigned char* smem, float tpass, int count, unsigned long long t_entry) {
  SolverState* sS = reinterpret_cast<SolverState*>(smem);
  double* sums = reinterpret_cast<double*>(smem + sizeof(SolverState));
  double* dots = sums + kMaxSlices * kHeadCols;
  int* flags = reinterpret_cast<int*>(dots + 5 * kSlots);
  __shared__ int s_go, s_dirty;
  __shared__ unsigned long long s_t[8];
  if (threadIdx.x == 0) s_t[0] = gtime();
  // the state's loads and the partial rows' loads are in flight together (one L2 round trip for both)
  constexpr int kStagePer = (kStateDoubles + 255) / 256;
  double stage[kStagePer];
  {
    const double* src = reinterpret_cast<const double*>(S);
#pragma unroll
    for (int q = 0; q < kStagePer; ++q) {
      const int k = (int)threadIdx.x + q * 256;
      stage[q] = (k < kStateDoubles) ? __ldcg(src + k) : 0.0;
    }
  }
  int slices = (count + kPairsPerSlice - 1) / kPairsPerSlice;
  if (slices < 1) slices = 1;
  for (int sl = 0; sl < slices; ++sl)
    reduce_head_rows(part + (int64_t)sl * nblocks * kHeadCols, nblocks, sums + sl * kHeadCols, kColVec + 3);
  {
    double* dst = reinterpret_cast<double*>(sS);
#pragma unroll
    for (int q = 0; q < kStagePer; ++q) {
      const int k = (int)threadIdx.x + q * 256;
      if (k < kStateDoubles) dst[k] = stage[q];
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) s_t[1] = gtime();
  const int pend = sS->pend, prev = sS->phase, n_iter = sS->lb.n_iter;
  if (threadIdx.x == 0) {
    s_t[2] = gtime();
    if (pend) {  // ---- finish the previous step ----
      double lsum = sums[kColLoss];
      if (sS->world > 1) lsum = (double)tl.tail[0] + (double)tl.tail[1];
      const double loss = (double)(float)(lsum / tl.p_total);  // fp32 mean as the reference sees it
      const double gtd = sums[kDotsPerSlice], gg = sums[kDotsPerSlice + 1], g1 = sums[kDotsPerSlice + 2];
      if (prev == PH_FRESH) fresh_apply(sS, loss, gg, g1);
      else if (prev != PH_MAT) {
        if (prev == PH_DIR) {  // the line-search init the vec kernel could not do (lbfgs.py:521-549)
          sS->gtd = (float)sums[kColVec]; sS->dd = sums[kColVec + 1]; sS->xx = sums[kColVec + 2];
          sS->dmax = (float)sums[kColVec + 3];
          ls_begin(sS->ls, sS->t_cur, sS->loss, (float)sums[kColVec], (float)sums[kColVec + 3]);
          sS->ls_active = 1;
        }
        ls_apply(sS, loss, gtd, gg, g1);
      }
      if (sS->error == MDE_E_COMM) sS->active = 0;
      int next = prev;
      bool end_of_iteration = false;
      if (prev == PH_FRESH) next = PH_DIR;
      else if (prev == PH_MAT) end_of_iteration = true;
      else if (sS->ls_active) next = PH_TRIAL;
      else if (sS->active) {
        if (sS->ls.t_accept == sS->t_eval) end_of_iteration = true;
        else next = PH_MAT;
      }
      if (end_of_iteration) {
        iter_end_body(sS, 0);
        next = sS->need_fresh ? PH_FRESH : PH_DIR;
        if (sS->active && sS->iter >= sS->iter_limit) { sS->active = 0; sS->paused = 1; }
      }
      set_phase(sS, next);
      if (next == PH_TRIAL) sS->t_cur = sS->ls.t;
      else if (next == PH_MAT) sS->t_cur = sS->ls.t_accept;
      sS->pend = 0;
    }
    s_go = (sS->active && sS->phase == PH_DIR) ? 1 : 0;
    s_dirty = (s_go || sS->lb.n_iter != n_iter) ? 1 : 0;  // (opt.reset() at the end of an iteration)
    s_t[3] = gtime();
  }
  __syncthreads();
  // ---- this step starts an iteration: history update + two-loop (the sums are those of THIS pass: valid because
  //      the accepted step is the one the pass assumed, or it ran with t_last after a pause / PH_MAT) ----
  if (s_go) {
    LbfgsState& B = sS->lb;
    if (threadIdx.x == 0) {
      // callback of LBFGS.step (optim.py:94-96): loss and ||X.grad||_F at the iteration start
      const int it = sS->iter;
      const double resid = (double)sqrtf((float)sS->gg);
      if (it < sS->max_stats) { sS->avg[it] = sS->loss; sS->resid[it] = resid; }
      sS->stop_after = (resid <= sS->eps) ? 1 : 0;
    }
    if ((int)threadIdx.x < count) {
      const int j = threadIdx.x;
      const double* b = sums + (j / kPairsPerSlice) * kHeadCols + 4 + 5 * (j % kPairsPerSlice);
      dots[j] = b[0]; dots[kSlots + j] = b[1]; dots[2 * kSlots + j] = b[2]; dots[3 * kSlots + j] = b[3];
      dots[4 * kSlots + j] = b[4];
    }
    __syncthreads();
    if (n_iter > 0) lbfgs_direction_block(B, dots, sums[0], sums[1], sums[2], sums[3], flags);
    else lbfgs_direction_block(B, dots, 0.0, 0.0, 0.0, 0.0, flags);
    __syncthreads();
    if (threadIdx.x == 64) s_t[4] = gtime();
    if (threadIdx.x < 32) {
      // column sums of d = cg g + sum_j cs_j S_j + cy_j Y_j from TRACKED column sums of the stored pairs
      // (S_c = t d_prev, Y_c = g - g_prev), lane j owning pair j.  These are rounding-level quantities (the gradient
      // of a translation-invariant objective sums to zero) and x's measured column mean corrects them every
      // iteration: fp32 shuffles, not an fp64 tree.
      const int lane = threadIdx.x;
      if (!flags[0] && flags[1] && lane < 4) {
        const int slot = B.order[B.count - 1];
        sS->cs_S[slot][lane] = (double)tpass * sS->cs_d[lane];
        sS->cs_Y[slot][lane] = sums[kColG + lane] - sS->cs_g[lane];
      }
      __syncwarp();
      const int q = (lane < B.count) ? B.order[lane] : 0;
      const float a = (lane < B.count) ? (float)B.cs[lane] : 0.0f, b = (lane < B.count) ? (float)B.cy[lane] : 0.0f;
      float v[4];
#pragma unroll
      for (int c = 0; c < 4; ++c) v[c] = a * (float)sS->cs_S[q][c] + b * (float)sS->cs_Y[q][c];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
#pragma unroll
        for (int c = 0; c < 4; ++c) v[c] += __shfl_xor_sync(kFull, v[c], o);
      }
      __syncwarp();
      if (lane < 4) {
        const float vl = lane == 0 ? v[0] : (lane == 1 ? v[1] : (lane == 2 ? v[2] : v[3]));
        const double cd = B.cg * sums[kColG + lane] + (double)vl;
        sS->cs_d[lane] = cd; sS->cs_g[lane] = sums[kColG + lane];
        sS->mu_d[lane] = (float)(cd * tl.inv_n);
        sS->mu_x[lane] = (float)(sums[kColX + lane] * tl.inv_n);
      }
    }
  }
  if ((threadIdx.x >> 5) == 1) {
    // (a different warp than the column sums: both run concurrently) first step length of a new iteration and the
    // 64-byte descriptor the next head kernel's blocks read
    const int lane = threadIdx.x & 31;
    double tc = sS->t_cur;
    if (s_go && sS->lb.n_iter == 1) {  // t = min(1, 1/||g||_1) * lr
      const float inv = 1.0f / (float)sS->g1;
      tc = (inv < 1.0f) ? (double)inv : 1.0;
    } else if (s_go) tc = 1.0;
    HeadDesc& h = sS->hd;
    h.order[lane] = (unsigned char)sS->lb.order[lane];
    if (lane == 0) {
      sS->t_cur = tc;
      sS->pend = sS->active ? 1 : 0;
      h.pend = sS->pend; h.phase = sS->phase; h.count = sS->lb.count; h.n_iter = sS->lb.n_iter; h.cand = sS->lb.cand;
      h.t_cur = (float)tc; h.t_last = (float)sS->t_last; h.pad = 0;
    }
  }
  if (threadIdx.x == 64 && s_go) {
    s_t[5] = gtime();
    sS->dbg[0] = t_entry;
    for (int k = 0; k < 6; ++k) sS->dbg[1 + k] = s_t[k];
  }
  __syncthreads();
  {
    double* dst = reinterpret_cast<double*>(S);
    const double* src = reinterpret_cast<const double*>(sS);
    const int n = s_dirty ? kStateDoubles : kLbOffsetDoubles;  // the history state only when it changed
    for (int k = threadIdx.x; k < n; k += blockDim.x) dst[k] = src[k];
  }
}

__global__ void __launch_bounds__(kVecThreads, 2)
step_head_kernel(SolverState* __restrict__ S, const float* __restrict__ g, const float* __restrict__ gprev,
                 const float* __restrict__ d, const float* __restrict__ X, float* __restrict__ Sb,
                 float* __restrict__ Yb, int64_t npad, int mcols, double* __restrict__ part,
                 const double* __restrict__ vpart, Tail tl) {
  if (off(&S->active)) return;
  __shared__ __align__(16) unsigned char raw[(kHeadSmemBytes + 15) / 16 * 16];  // warp sums, then the scalar stage
  static_assert(sizeof(raw) >= sizeof(float) * kHeadAcc * (kVecThreads / 32), "warp sums must fit");
  static_assert(kHeadAcc == 66, "the transposing butterfly below is written for 64 + 2 accumulators");
  __shared__ const float* sp[kPairsPerSlice];
  __shared__ const float* yp[kPairsPerSlice];
  const unsigned long long t_entry = gtime();
  const int slice = blockIdx.y;
  // one round trip: the 64-byte descriptor the previous epilogue left (same address for every thread)
  const int4 h0 = __ldcg(reinterpret_cast<const int4*>(&S->hd));
  const int4 h1 = __ldcg(reinterpret_cast<const int4*>(&S->hd) + 1);
  const uint4 h2 = __ldcg(reinterpret_cast<const uint4*>(&S->hd) + 2);
  const uint4 h3 = __ldcg(reinterpret_cast<const uint4*>(&S->hd) + 3);
  const int pend = h0.x, prev = h0.y, count = h0.z, n_iter0 = h0.w;
  const bool want_grad = pend && prev != PH_MAT && slice == 0;
  const bool want_hist = (n_iter0 != 0) && !(pend && prev == PH_FRESH) && (slice == 0 || slice * kPairsPerSlice < count);
  const bool spec = pend && (prev == PH_DIR || prev == PH_TRIAL);
  const float t = spec ? __int_as_float(h1.y) : __int_as_float(h1.z);
  // warp 7's share of the previous launches' partials: issued now, used after the pass
  double pre_loss = 0.0, pre_vec = 0.0;
  if ((threadIdx.x >> 5) == 7 && want_grad) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x + lane * (int)gridDim.x;
    if (j < tl.nl) pre_loss = __ldcg(tl.lpart + j);
    if (lane < 4 && prev == PH_DIR) pre_vec = __ldcg(vpart + (int64_t)blockIdx.x * 4 + lane);
  }
  float acc[kHeadAcc];
#pragma unroll
  for (int k = 0; k < kHeadAcc; ++k) acc[k] = 0.0f;
  if (want_grad || want_hist || slice == 0) {
    float* sc = Sb + (int64_t)h1.x * npad;
    float* yc = Yb + (int64_t)h1.x * npad;
    if (threadIdx.x < kPairsPerSlice) {
      const int lj = slice * kPairsPerSlice + threadIdx.x;
      const unsigned ow[8] = {h2.x, h2.y, h2.z, h2.w, h3.x, h3.y, h3.z, h3.w};
      unsigned word = ow[0];
#pragma unroll
      for (int q = 1; q < 8; ++q) if ((lj >> 2) == q) word = ow[q];
      const int q = (lj < count && lj < 32) ? (int)((word >> (8 * (lj & 3))) & 0xffu) : 0;
      sp[threadIdx.x] = Sb + (int64_t)q * npad;
      yp[threadIdx.x] = Yb + (int64_t)q * npad;
    }
    __syncthreads();
    int nval = want_hist ? count - slice * kPairsPerSlice : 0;
    if (nval > kPairsPerSlice) nval = kPairsPerSlice;
    const int64_t n4 = npad >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
      const float4 G = reinterpret_cast<const float4*>(g)[i];
      const float gv[4] = {G.x, G.y, G.z, G.w};
      if (slice == 0) {
        const float4 Xv = reinterpret_cast<const float4*>(X)[i];
        // column sums (rows are m floats; 4 % m == 0 so element q of a float4 belongs to column q % m)
        if (mcols == 1) {
          acc[kColG] += (G.x + G.y) + (G.z + G.w); acc[kColX] += (Xv.x + Xv.y) + (Xv.z + Xv.w);
        } else if (mcols == 2) {
          acc[kColG] += G.x + G.z; acc[kColG + 1] += G.y + G.w; acc[kColX] += Xv.x + Xv.z; acc[kColX + 1] += Xv.y + Xv.w;
        } else if (mcols == 4) {
          acc[kColG] += G.x; acc[kColG + 1] += G.y; acc[kColG + 2] += G.z; acc[kColG + 3] += G.w;
          acc[kColX] += Xv.x; acc[kColX + 1] += Xv.y; acc[kColX + 2] += Xv.z; acc[kColX + 3] += Xv.w;
        }
      }
      if (!(want_grad || want_hist)) continue;
      const float4 P = reinterpret_cast<const float4*>(gprev)[i];
      const float4 D = reinterpret_cast<const float4*>(d)[i];
      const float dv[4] = {D.x, D.y, D.z, D.w};
      const float yv[4] = {G.x - P.x, G.y - P.y, G.z - P.z, G.w - P.w};
      const float sv[4] = {D.x * t, D.y * t, D.z * t, D.w * t};
      if (want_grad) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          acc[kDotsPerSlice] += gv[q] * dv[q];
          acc[kDotsPerSlice + 1] += gv[q] * gv[q];
          acc[kDotsPerSlice + 2] += fabsf(gv[q]);
        }
      }
      if (want_hist && slice == 0) {
        reinterpret_cast<float4*>(yc)[i] = make_float4(yv[0], yv[1], yv[2], yv[3]);
        reinterpret_cast<float4*>(sc)[i] = make_float4(sv[0], sv[1], sv[2], sv[3]);
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          acc[0] += yv[q] * sv[q]; acc[1] += yv[q] * yv[q];
          acc[2] += sv[q] * gv[q]; acc[3] += yv[q] * gv[q];
        }
      }
#pragma unroll
      for (int j = 0; j < kPairsPerSlice; ++j) {
        if (j < nval) {
          const float4 A = reinterpret_cast<const float4*>(sp[j])[i];
          const float4 B = reinterpret_cast<const float4*>(yp[j])[i];
          const float av[4] = {A.x, A.y, A.z, A.w};
          const float bv[4] = {B.x, B.y, B.z, B.w};
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            acc[4 + 5 * j + 0] += av[q] * yv[q];
            acc[4 + 5 * j + 1] += bv[q] * yv[q];
            acc[4 + 5 * j + 2] += sv[q] * bv[q];
            acc[4 + 5 * j + 3] += av[q] * gv[q];
            acc[4 + 5 * j + 4] += bv[q] * gv[q];
          }
        }
      }
    }
  }
  {
    // Block reduction of the 66 per-thread accumulators.  Warp level: a transposing butterfly -- at the level with
    // lane distance o a lane keeps half of its values and sends the other half, so 64 values cost 62 shuffles
    // (a plain butterfly: 320) and lane L ends with the warp totals of accumulators idx(L) and idx(L) + 1.  Block
    // level: 8 warps through shared memory.  fp32 inside the block (its 256 per-thread partials are fp32 anyway),
    // double across blocks.  The summation order is fixed.
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    float (*wsum)[kHeadAcc] = reinterpret_cast<float (*)[kHeadAcc]>(raw);
#define MDE_TR_LEVEL(N, O)                                                              \
    _Pragma("unroll") for (int i = 0; i < (N); ++i) {                                   \
      const bool hi = (lane & (O)) != 0;                                                \
      const float a_ = acc[i], b_ = acc[i + (N)];                                       \
      acc[i] = (hi ? b_ : a_) + __shfl_xor_sync(kFull, hi ? a_ : b_, (O));              \
    }
    MDE_TR_LEVEL(32, 16) MDE_TR_LEVEL(16, 8) MDE_TR_LEVEL(8, 4) MDE_TR_LEVEL(4, 2) MDE_TR_LEVEL(2, 1)
#undef MDE_TR_LEVEL
    const int idx = ((lane & 16) ? 32 : 0) | ((lane & 8) ? 16 : 0) | ((lane & 4) ? 8 : 0) | ((lane & 2) ? 4 : 0) |
                    ((lane & 1) ? 2 : 0);
    const float x64 = warp_sum(acc[64]);
    wsum[w][idx] = acc[0]; wsum[w][idx + 1] = acc[1];
    if (lane == 0) { wsum[w][64] = x64; wsum[w][65] = 0.0f; }
    __syncthreads();
    double* o = part + ((int64_t)slice * gridDim.x + blockIdx.x) * kHeadCols;
    if (threadIdx.x < kHeadAcc) {
      float s0 = 0.0f, s1 = 0.0f;
#pragma unroll
      for (int q = 0; q < kVecThreads / 32; q += 2) { s0 += wsum[q][threadIdx.x]; s1 += wsum[q + 1][threadIdx.x]; }
      o[threadIdx.x] = (double)(s0 + s1);
    }
    // the row also carries this block's share of the pending evaluation's loss partials (scatter launch) and of
    // the pending PH_DIR step's vec partials (loaded at the top), so that the epilogue reduces ONE array
    if (w == 7) {
      double ls = pre_loss;
      if (want_grad) {
        for (int j = blockIdx.x + (lane + 32) * (int)gridDim.x; j < tl.nl; j += 32 * (int)gridDim.x) ls += __ldcg(tl.lpart + j);
        ls = warp_sum(ls);
      }
      if (lane == 0) o[kColLoss] = ls;
      if (lane < 4) o[kColVec + lane] = pre_vec;
      if (lane == 4) o[kHeadCols - 1] = 0.0;
    }
  }
  if (last_block_done(&S->tickets[0])) step_head_body(S, part, gridDim.x, tl, raw, t, count, t_entry);
}

// the vector kernel of a late-epilogue step (see above).  `gz` is the buffer the scatter kernel adds into: g itself
// on one GPU (zeroed AFTER this thread has read its elements), the peer-visible partial buffer on several.
__global__ void __launch_bounds__(kVecThreads)
step_vec_kernel(SolverState* __restrict__ S, const float* g, float* __restrict__ gprev, float* __restrict__ d,
                float* __restrict__ X, float* __restrict__ xinit, const float* __restrict__ Sb,
                const float* __restrict__ Yb, int64_t npad, int64_t nvalid, int center_m, float* gz,
                const Comm* __restrict__ comm, double* __restrict__ vpart) {
  if (off(&S->active)) return;
  const int ph = S->phase;  // written by the head kernel's epilogue
  if (blockIdx.x == 0 && threadIdx.x == 0 && ph == PH_DIR) S->dbg[7] = gtime();
  const bool mat = ph == PH_MAT, dir = ph == PH_DIR, move = ph != PH_FRESH;
  if (comm != nullptr && !mat) comm_wait_readers_fwd(comm, &S->error);  // gz is the peer-visible partial buffer
  const float t = (float)S->t_cur;
  float mu[4] = {0.f, 0.f, 0.f, 0.f};
  if (center_m == 1) { float v = S->mu_x[0] + t * S->mu_d[0]; mu[0] = mu[1] = mu[2] = mu[3] = v; }
  else if (center_m == 2) {
    float v0 = S->mu_x[0] + t * S->mu_d[0], v1 = S->mu_x[1] + t * S->mu_d[1];
    mu[0] = mu[2] = v0; mu[1] = mu[3] = v1;
  } else if (center_m == 4) {
#pragma unroll
    for (int c = 0; c < 4; ++c) mu[c] = S->mu_x[c] + t * S->mu_d[c];
  }
  __shared__ float cs[kMaxMemory], cy[kMaxMemory];
  __shared__ const float* ps[kMaxMemory];
  __shared__ const float* py[kMaxMemory];
  const int count = dir ? S->lb.count : 0;
  const float cg = (float)S->lb.cg;
  if ((int)threadIdx.x < count) {
    cs[threadIdx.x] = (float)S->lb.cs[threadIdx.x];
    cy[threadIdx.x] = (float)S->lb.cy[threadIdx.x];
    const int q = S->lb.order[threadIdx.x];
    ps[threadIdx.x] = Sb + (int64_t)q * npad;
    py[threadIdx.x] = Yb + (int64_t)q * npad;
  }
  __syncthreads();
  double acc[3] = {0.0, 0.0, 0.0};
  float fa[3] = {0.0f, 0.0f, 0.0f};
  float mx = 0.0f;
  int cnt = 0;
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4 + 1; i += stride) {
    if (move && i < n4) {
      float4 A, D;
      if (dir) {
        const float4 G = reinterpret_cast<const float4*>(g)[i];
        A = reinterpret_cast<const float4*>(X)[i];
        float r[4] = {cg * G.x, cg * G.y, cg * G.z, cg * G.w};
        for (int j = 0; j < count; ++j) {
          const float4 Sv = reinterpret_cast<const float4*>(ps[j])[i];
          const float4 Yv = reinterpret_cast<const float4*>(py[j])[i];
          r[0] += cs[j] * Sv.x + cy[j] * Yv.x; r[1] += cs[j] * Sv.y + cy[j] * Yv.y;
          r[2] += cs[j] * Sv.z + cy[j] * Yv.z; r[3] += cs[j] * Sv.w + cy[j] * Yv.w;
        }
        D = make_float4(r[0], r[1], r[2], r[3]);
        reinterpret_cast<float4*>(d)[i] = D;
        reinterpret_cast<float4*>(gprev)[i] = G;
        reinterpret_cast<float4*>(xinit)[i] = A;
        fa[0] += G.x * r[0] + G.y * r[1] + G.z * r[2] + G.w * r[3];
        fa[1] += r[0] * r[0] + r[1] * r[1] + r[2] * r[2] + r[3] * r[3];
        fa[2] += A.x * A.x + A.y * A.y + A.z * A.z + A.w * A.w;
        mx = fmaxf(mx, fmaxf(fmaxf(fabsf(r[0]), fabsf(r[1])), fmaxf(fabsf(r[2]), fabsf(r[3]))));
        if (++cnt == 16) {
#pragma unroll
          for (int k = 0; k < 3; ++k) { acc[k] += (double)fa[k]; fa[k] = 0.0f; }
          cnt = 0;
        }
      } else {
        A = reinterpret_cast<const float4*>(xinit)[i];
        D = reinterpret_cast<const float4*>(d)[i];
      }
      float4 R = make_float4(fmaf(t, D.x, A.x) - mu[0], fmaf(t, D.y, A.y) - mu[1], fmaf(t, D.z, A.z) - mu[2],
                             fmaf(t, D.w, A.w) - mu[3]);
      if (center_m != 0 && 4 * i + 3 >= nvalid) {  // keep the zero padding behind the last row
        if (4 * i + 0 >= nvalid) R.x = 0.f;
        if (4 * i + 1 >= nvalid) R.y = 0.f;
        if (4 * i + 2 >= nvalid) R.z = 0.f;
        if (4 * i + 3 >= nvalid) R.w = 0.f;
      }
      reinterpret_cast<float4*>(X)[i] = R;
    }
    if (!mat) reinterpret_cast<float4*>(gz)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (dir) {
#pragma unroll
    for (int k = 0; k < 3; ++k) acc[k] += (double)fa[k];
    __shared__ double sm[3 * 32];
    __shared__ float smx[32];
    block_sum<3>(acc, sm);
    mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) smx[threadIdx.x >> 5] = mx;
    __syncthreads();
    if (threadIdx.x == 0) {
      float m2 = 0.0f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) m2 = fmaxf(m2, smx[w]);
      double* o = vpart + (int64_t)blockIdx.x * 4;
      o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2]; o[3] = (double)m2;
    }
  }
}

// mode 2: (re)arm the solver for iterations up to `limit`
__global__ void resume_kernel(SolverState* __restrict__ S, int limit) {
  if (threadIdx.x != 0) return;
  S->iter_limit = limit;
  if (S->paused && S->iter < limit) { S->paused = 0; S->active = 1; }
  else if (S->active && S->iter >= limit) { S->active = 0; S->paused = 1; }
  set_phase(S, S->phase);
}

// mode 2: the axpy of a step.  PH_DIR / PH_TRIAL: trial point x_init + t d (and g = 0 for the scatter that
// follows); PH_MAT: accepted point x_init + t_accept d; PH_FRESH: only g = 0.  Centered with m in {1,2,4}
// is applied on the fly like trial_axpy_kernel.
__global__ void __launch_bounds__(kVecThreads)
step_axpy_kernel(SolverState* __restrict__ S, const float* __restrict__ xinit, const float* __restrict__ d,
                 float* __restrict__ X, int64_t npad, int64_t nvalid, int center_m, float* __restrict__ gz,
                 const Comm* __restrict__ comm) {
  if (off(&S->active)) return;
  const bool mat = S->g_mat != 0;
  if (comm != nullptr && !mat) comm_wait_readers_fwd(comm, &S->error);  // gz is the peer-visible partial buffer
  const bool move = S->g_proj != 0;  // every phase but PH_FRESH
  if (move && !mat && off(&S->ls_active)) return;
  const float t = mat ? (float)S->ls.t_accept : (float)S->ls.t;
  float mu[4] = {0.f, 0.f, 0.f, 0.f};
  if (center_m == 1) { float v = S->mu_x[0] + t * S->mu_d[0]; mu[0] = mu[1] = mu[2] = mu[3] = v; }
  else if (center_m == 2) {
    float v0 = S->mu_x[0] + t * S->mu_d[0], v1 = S->mu_x[1] + t * S->mu_d[1];
    mu[0] = mu[2] = v0; mu[1] = mu[3] = v1;
  } else if (center_m == 4) {
#pragma unroll
    for (int c = 0; c < 4; ++c) mu[c] = S->mu_x[c] + t * S->mu_d[c];
  }
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4 + 1; i += stride) {
    if (move && i < n4) {
      float4 A = reinterpret_cast<const float4*>(xinit)[i];
      float4 D = reinterpret_cast<const float4*>(d)[i];
      float4 R = make_float4(fmaf(t, D.x, A.x) - mu[0], fmaf(t, D.y, A.y) - mu[1], fmaf(t, D.z, A.z) - mu[2],
                             fmaf(t, D.w, A.w) - mu[3]);
      if (center_m != 0 && 4 * i + 3 >= nvalid) {  // keep the zero padding behind the last row
        if (4 * i + 0 >= nvalid) R.x = 0.f;
        if (4 * i + 1 >= nvalid) R.y = 0.f;
        if (4 * i + 2 >= nvalid) R.z = 0.f;
        if (4 * i + 3 >= nvalid) R.w = 0.f;
      }
      reinterpret_cast<float4*>(X)[i] = R;
    }
    if (!mat) reinterpret_cast<float4*>(gz)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__global__ void init_state_kernel(SolverState* S, double eps, int memory, int max_stats, int world,
                                  double* avg, double* resid, double* pct, double* steplen) {
  if (threadIdx.x != 0) return;
  S->active = 1; S->converged = 0; S->iter = 0; S->error = 0; S->need_fresh = 1; S->ls_active = 0;
  S->stop_after = 0; S->pad0 = 0; S->eps = eps; S->loss = 0.0; S->gg = 0.0; S->g1 = 0.0; S->gtd = 0.0f;
  S->dmax = 0.0f; S->dd = 0.0; S->xx = 0.0; S->t_last = 0.0; S->t_eval = 0.0; S->func_evals = 0;
  S->max_stats = max_stats; S->world = world;
  S->paused = 0; S->iter_limit = max_stats; S->pend = 0;
  S->t_cur = 0.0;
  for (int c = 0; c < 4; ++c) { S->cs_g[c] = 0.0; S->cs_d[c] = 0.0; S->mu_x[c] = 0.0f; S->mu_d[c] = 0.0f; }
  for (int q = 0; q < kSlots; ++q) for (int c = 0; c < 4; ++c) { S->cs_S[q][c] = 0.0; S->cs_Y[q][c] = 0.0; }
  set_phase(S, PH_FRESH);  // mode 2 (sets need_fresh = 1 as well)
  for (int k = 0; k < 4; ++k) S->tickets[k] = 0u;
  S->avg = avg; S->resid = resid; S->pct = pct; S->steplen = steplen;
  lbfgs_reset(S->lb, memory);
  ls_begin(S->ls, 0.0, 0.0, 0.0f, 0.0f);
  S->ls.phase = LS_DONE;
  fill_head_desc(S);
}

int vec_blocks(int64_t n4) {
  int64_t nb = (n4 + kVecThreads - 1) / kVecThreads;
  if (nb < 1) nb = 1;
  if (nb > kVecBlocks) nb = kVecBlocks;
  return (int)nb;
}

}  // namespace

struct mde_solver {
  const mde_edges* edges = nullptr;
  int64_t n = 0, N = 0, npad = 0;
  int m = 0;
  mde_solver_opts_t opts{};
  SolverState* S = nullptr;          // device
  int* status_host = nullptr;        // pinned, kStatusInts ints
  float *X = nullptr, *xinit = nullptr, *d = nullptr, *g = nullptr, *gprev = nullptr, *Sb = nullptr, *Yb = nullptr;
  float* gpart = nullptr;            // mode 2, multi-GPU: this rank's partial [gradient | loss] before the all-reduce
  double *dpart = nullptr;           // dot partials
  double *vpart = nullptr;           // late-epilogue steps: (g.d, d.d, X.X, max|d|) partials of the vec kernel
  double *stats = nullptr;           // 4 * max_iter doubles
  void* projws = nullptr;
  ProjWs pw{};
  int fuse = 1;                      // scalar epilogues run in the last block of the vector kernels
  int center_m = 0;                  // {1,2,4}: Centered projection fused into the trial axpy
  int nl = 0;                        // loss-partial blocks of the distortion launch
  int nvb = 0;                       // vector-pass blocks
  int host_need_fresh = 1;
  int host_active = 0;
  int host_evals = 0;                // func_evals already accounted in the launch counter (mode 1)
  mde_allreduce_fn allreduce = nullptr;
  void* allreduce_user = nullptr;
  // peer-memory all-reduce (world_size > 1): one cudaMalloc region [partial buffer | flags | epoch | ticket],
  // exported with cudaIpc, the peers' regions mapped by mde_solver_comm_connect
  void* comm_region = nullptr;
  int64_t comm_bytes = 0, comm_flags_off = 0, comm_g_off = 0, comm_recv_off = 0, comm_tails_off = 0, comm_slot_floats = 0;
  int comm_pull = 0;                 // read-based two-shot instead of the push kernels (A/B switch)
  Comm comm{};
  Comm* comm_dev = nullptr;
  int comm_connected = 0;
  void* peer_base[kMaxWorld] = {nullptr};
  int64_t* anchors = nullptr;
  float* anchor_values = nullptr;
  // mode 1: one CUDA graph per iteration with an IF node (fresh evaluation) and a WHILE node (trials)
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  // the same iteration chained `unroll` times in one graph: one graph launch per `unroll` iterations
  cudaGraph_t graph_u = nullptr;
  cudaGraphExec_t graph_exec_u = nullptr;
  int unroll = 1;
  // mode 2: flat step graphs (one step / steps_per_graph steps), no conditional nodes
  int steps_per_graph = 8;           // MDE_B200_STEPS (1..64)
  int late = 0;                      // mode 2: evaluation bookkeeping rides in the next step's head kernel (MDE_B200_LATE=0: off)
  cudaGraph_t step_graph = nullptr, steps_graph = nullptr;
  cudaGraphExec_t step_exec = nullptr, steps_exec = nullptr;
  int step_kernels = 0;              // kernel nodes per step
  int host_iter = 0;                 // iterations completed (last status read)
  int cur_max_iter = 0;              // iteration cap of the current solve (<= opts.max_iter)
  cudaStream_t cap_stream = nullptr, cap_stream2 = nullptr;
  cudaGraphConditionalHandle h_if = 0, h_while = 0, h_if_next = 0;  // capture-time only
  int graph_kernels_fixed = 0, graph_kernels_trial = 0, graph_kernels_fresh = 0;
};

namespace {

int read_status(mde_solver* s, cudaStream_t st) {
  MDE_CUDA_TRY(cudaMemcpyAsync(s->status_host, s->S, kStatusInts * sizeof(int), cudaMemcpyDeviceToHost, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// project the iterate onto the constraint set (project_callback, lbfgs.py:368-372)
int enqueue_project(mde_solver* s, cudaStream_t st) {
  const int* act = &s->S->active;
  switch (s->opts.constraint) {
    case MDE_CONSTRAINT_CENTERED:
      if (s->center_m) return 0;  // already applied by trial_axpy_kernel
      return enqueue_project_centered(s->X, s->n, s->m, s->pw, act, st);
    case MDE_CONSTRAINT_STANDARDIZED: return enqueue_project_standardized(s->X, s->n, s->m, s->pw, act, st);
    case MDE_CONSTRAINT_ANCHORED: {
      int64_t tot = s->opts.n_anchors * s->m;
      if (tot > 0) {
        anchor_rows_kernel<<<(int)((tot + 255) / 256), 256, 0, st>>>(act, s->X, s->anchors, s->anchor_values,
                                                                    s->opts.n_anchors, s->m);
        MDE_LAUNCH_CHECK();
      }
      return 0;
    }
  }
  return MDE_E_INVALID;
}

// closure: value_and_grad at s->X (optim.py:100-105); `flag` gates the kernels
Tail make_tail(mde_solver* s, int mode) {
  Tail tl;
  tl.fuse = s->fuse; tl.mode = mode;
  tl.lpart = loss_partials_ptr(s->edges); tl.nl = s->nl; tl.tail = s->g + s->npad;
  tl.p_total = (double)edges_p_total(s->edges); tl.n_rows = s->n; tl.inv_n = 1.0 / (double)s->n; tl.h_while = s->h_while;
  return tl;
}

int enqueue_eval(mde_solver* s, const int* flag, bool zero_g, int tail_mode, cudaStream_t st, bool with_dots = true) {
  // several GPUs: scatter into this rank's partial buffer (peer-visible), then all-reduce into g
  const bool multi = s->opts.world_size > 1;
  const bool staged = multi && s->opts.mode == 2;  // (the peer-memory path exists in mode 2 only)
  float* target = staged ? s->gpart : s->g;
  if (zero_g) {
    const int64_t n4 = (s->npad + 4) >> 2;  // gradient + (hi, lo) tail
    zero_kernel<<<vec_blocks(n4), kVecThreads, 0, st>>>(flag, target, n4);
    MDE_LAUNCH_CHECK();
  }
  int rc = distortion_fused_flag(s->edges, s->X, s->m, target, &s->nl, flag, st);
  if (rc) return rc;
  if (multi) {
    pack_loss_kernel<<<1, 256, 0, st>>>(flag, loss_partials_ptr(s->edges), s->nl, target + s->npad);
    MDE_LAUNCH_CHECK();
    if (s->comm_connected) {
      const int64_t n4 = s->npad >> 2;
      int nb = (int)((n4 + kCommThreads - 1) / kCommThreads);
      if (nb > kNumSMs) nb = kNumSMs;  // one resident 512-thread block per SM (84-100 registers): a single wave
      if (nb < 1) nb = 1;
      if ((s->npad + 4) * (int64_t)sizeof(float) <= kOneShotBytes) {
        allreduce_kernel<0><<<nb, kCommThreads, 0, st>>>(flag, s->comm, s->g, s->npad, &s->S->error);
        MDE_LAUNCH_CHECK();
      } else if (s->comm_pull) {  // MDE_B200_ALLREDUCE=pull: read-based reduce-scatter + all-gather (A/B)
        allreduce_kernel<1><<<nb, kCommThreads, 0, st>>>(flag, s->comm, s->g, s->npad, &s->S->error);
        MDE_LAUNCH_CHECK();
        allreduce_kernel<2><<<nb, kCommThreads, 0, st>>>(flag, s->comm, s->g, s->npad, &s->S->error);
        MDE_LAUNCH_CHECK();
      } else {
        allreduce_push_kernel<0><<<nb, kCommThreads, 0, st>>>(flag, s->comm, s->npad, &s->S->error);
        MDE_LAUNCH_CHECK();
        allreduce_push_kernel<1><<<nb, kCommThreads, 0, st>>>(flag, s->comm, s->npad, &s->S->error);
        MDE_LAUNCH_CHECK();
        allreduce_push_kernel<2><<<1, 32, 0, st>>>(flag, s->comm, s->npad, &s->S->error);
        MDE_LAUNCH_CHECK();
      }
    } else {
      // host hook (an NCCL all-reduce enqueued by the caller between two kernels): not graph-capturable
      if (!s->allreduce) return MDE_E_INVALID;
      rc = s->allreduce(s->allreduce_user, target, s->npad + 4, (void*)st);
      if (rc) return rc;
      if (staged) {
        const int64_t n4 = (s->npad + 4) >> 2;
        gated_copy_kernel<<<vec_blocks(n4), kVecThreads, 0, st>>>(flag, s->gpart, s->g, n4);
        MDE_LAUNCH_CHECK();
      }
    }
  }
  const int* act = flag;
  if (s->opts.constraint == MDE_CONSTRAINT_STANDARDIZED) {
    rc = enqueue_tangent_standardized(s->X, s->g, s->n, s->m, s->pw, act, st);
    if (rc) return rc;
  } else if (s->opts.constraint == MDE_CONSTRAINT_ANCHORED) {
    int64_t tot = s->opts.n_anchors * s->m;
    if (tot > 0) {
      anchor_rows_kernel<<<(int)((tot + 255) / 256), 256, 0, st>>>(act, s->g, s->anchors, nullptr,
                                                                  s->opts.n_anchors, s->m);
      MDE_LAUNCH_CHECK();
    }
  }
  if (!with_dots) return 0;  // late-epilogue steps: the next step's head kernel computes them
  Tail tl = make_tail(s, tail_mode);
  grad_dots_kernel<<<s->nvb, kVecThreads, 0, st>>>(flag, s->g, s->d, s->npad, s->dpart, s->S, tl);
  MDE_LAUNCH_CHECK();
  return 0;
}

int enqueue_fresh(mde_solver* s, cudaStream_t st) {
  int rc = enqueue_eval(s, &s->S->need_fresh, true, 2, st);
  if (rc) return rc;
  if (!s->fuse) {
    fresh_finish_kernel<<<1, 256, 0, st>>>(s->S, loss_partials_ptr(s->edges), s->nl, s->g + s->npad, s->dpart,
                                           s->nvb, (double)edges_p_total(s->edges));
    MDE_LAUNCH_CHECK();
  }
  return 0;
}

int enqueue_direction(mde_solver* s, cudaStream_t st, const int* gate = nullptr) {
  int slices = (s->opts.memory_size + kPairsPerSlice - 1) / kPairsPerSlice;
  dim3 grid(s->nvb, slices);
  Tail tl = make_tail(s, 0);
  lbfgs_dots_kernel<<<grid, kVecThreads, 0, st>>>(s->S, s->g, s->gprev, s->d, s->Sb, s->Yb, s->npad, s->dpart, tl,
                                                  gate);
  MDE_LAUNCH_CHECK();
  if (!s->fuse) {
    direction_scalar_kernel<<<1, 256, 0, st>>>(s->S, s->dpart, s->nvb);
    MDE_LAUNCH_CHECK();
  }
  direction_apply_kernel<<<s->nvb, kVecThreads, 0, st>>>(s->S, s->g, s->gprev, s->d, s->X, s->xinit, s->Sb,
                                                         s->Yb, s->npad, s->dpart, s->center_m, tl, gate);
  MDE_LAUNCH_CHECK();
  if (!s->fuse) {
    ls_init_kernel<<<1, 256, 0, st>>>(s->S, s->dpart, s->nvb, s->n, s->h_while);
    MDE_LAUNCH_CHECK();
  }
  return 0;
}

int enqueue_trial(mde_solver* s, cudaStream_t st) {
  trial_axpy_kernel<false><<<s->nvb, kVecThreads, 0, st>>>(s->S, s->xinit, s->d, s->X, s->npad, s->N, s->center_m, s->g, 0, 0);
  MDE_LAUNCH_CHECK();
  int rc = enqueue_project(s, st);
  if (rc) return rc;
  rc = enqueue_eval(s, &s->S->ls_active, false, 1, st);
  if (rc) return rc;
  if (!s->fuse) {
    ls_update_kernel<<<1, 256, 0, st>>>(s->S, loss_partials_ptr(s->edges), s->nl, s->g + s->npad, s->dpart, s->nvb,
                                        (double)edges_p_total(s->edges), s->h_while);
    MDE_LAUNCH_CHECK();
  }
  return 0;
}

int enqueue_finish(mde_solver* s, cudaStream_t st) {
  // iter_end may ride in the axpy's last block only when no projection kernel follows (it can clear `active`)
  const int fuse_end = (s->fuse && s->opts.constraint == MDE_CONSTRAINT_CENTERED && s->center_m) ? 1 : 0;
  trial_axpy_kernel<true><<<s->nvb, kVecThreads, 0, st>>>(s->S, s->xinit, s->d, s->X, s->npad, s->N, s->center_m,
                                                          nullptr, fuse_end, s->h_if_next);
  MDE_LAUNCH_CHECK();
  int rc = enqueue_project(s, st);
  if (rc) return rc;
  if (!fuse_end) {
    iter_end_kernel<<<1, 32, 0, st>>>(s->S, s->h_if_next);
    MDE_LAUNCH_CHECK();
  }
  return 0;
}

// mode 2: one step (see step_end_body).  Every kernel is gated on the device; the chain has no host decision.
int enqueue_step(mde_solver* s, cudaStream_t st) {
  SolverState* S = s->S;
  int rc = 0;
  if (s->late) {
    int slices = (s->opts.memory_size + kPairsPerSlice - 1) / kPairsPerSlice;
    dim3 grid(s->nvb, slices);
    Tail tl = make_tail(s, 3);
    step_head_kernel<<<grid, kVecThreads, 0, st>>>(S, s->g, s->gprev, s->d, s->X, s->Sb, s->Yb, s->npad, s->center_m,
                                                   s->dpart, s->vpart, tl);
    MDE_LAUNCH_CHECK();
    step_vec_kernel<<<s->nvb, kVecThreads, 0, st>>>(S, s->g, s->gprev, s->d, s->X, s->xinit, s->Sb, s->Yb, s->npad,
                                                    s->N, s->center_m, s->opts.world_size > 1 ? s->gpart : s->g,
                                                    s->comm_connected ? s->comm_dev : nullptr, s->vpart);
    MDE_LAUNCH_CHECK();
  } else {
    if ((rc = enqueue_direction(s, st, &S->g_dir))) return rc;
    step_axpy_kernel<<<s->nvb, kVecThreads, 0, st>>>(S, s->xinit, s->d, s->X, s->npad, s->N, s->center_m,
                                                     s->opts.world_size > 1 ? s->gpart : s->g,
                                                     s->comm_connected ? s->comm_dev : nullptr);
    MDE_LAUNCH_CHECK();
  }
  switch (s->opts.constraint) {  // retraction of the moved iterate (project_callback, lbfgs.py:368-372)
    case MDE_CONSTRAINT_CENTERED:
      if (!s->center_m && (rc = enqueue_project_centered(s->X, s->n, s->m, s->pw, &S->g_proj, st))) return rc;
      break;
    case MDE_CONSTRAINT_STANDARDIZED:
      if ((rc = enqueue_project_standardized(s->X, s->n, s->m, s->pw, &S->g_proj, st))) return rc;
      break;
    case MDE_CONSTRAINT_ANCHORED: {
      const int64_t tot = s->opts.n_anchors * s->m;
      if (tot > 0) {
        anchor_rows_kernel<<<(int)((tot + 255) / 256), 256, 0, st>>>(&S->g_proj, s->X, s->anchors, s->anchor_values,
                                                                    s->opts.n_anchors, s->m);
        MDE_LAUNCH_CHECK();
      }
      break;
    }
    default: return MDE_E_INVALID;
  }
  return enqueue_eval(s, &S->g_eval, false, 3, st, !s->late);
}

int build_step_graph(mde_solver* s, int steps, cudaGraph_t* graph_out, cudaGraphExec_t* exec_out) {
#define GTRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return (int)_e; } while (0)
  if (!s->cap_stream) GTRY(cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
  const unsigned long long l0 = g_launch_count;
  if (s->late && s->nl == 0) {
    // the head kernel of a step reads the loss partials of the PREVIOUS step's scatter launch: their count is
    // known once one evaluation has been enqueued, so capture one throw-away step first
    cudaGraph_t tmp = nullptr;
    GTRY(cudaStreamBeginCapture(s->cap_stream, cudaStreamCaptureModeRelaxed));
    int rc0 = enqueue_step(s, s->cap_stream);
    cudaError_t e0 = cudaStreamEndCapture(s->cap_stream, &tmp);
    if (tmp) cudaGraphDestroy(tmp);
    if (rc0) return rc0;
    GTRY(e0);
    g_launch_count = l0;
  }
  GTRY(cudaStreamBeginCapture(s->cap_stream, cudaStreamCaptureModeRelaxed));
  int rc = 0;
  for (int k = 0; k < steps && !rc; ++k) rc = enqueue_step(s, s->cap_stream);
  cudaError_t e = cudaStreamEndCapture(s->cap_stream, graph_out);
  if (rc) return rc;
  GTRY(e);
  GTRY(cudaGraphInstantiate(exec_out, *graph_out, 0));
  s->step_kernels = (int)(g_launch_count - l0) / steps;
  g_launch_count = l0;  // capture enqueued nothing; launches are counted per graph launch
  return 0;
#undef GTRY
}

// One iteration as a CUDA graph:
//   fresh_gate -> IF(need_fresh){ evaluate at X } -> direction (P1,S1,P2,S2) -> WHILE(ls_active){ trial }
//   -> accepted step + projection + iter_end.
// The conditional handles are written on the device (cudaGraphSetConditional), so the host never reads
// a scalar during an iteration.
int build_iteration_graph(mde_solver* s, int copies, cudaGraph_t* graph_out, cudaGraphExec_t* exec_out) {
#define GTRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return (int)_e; } while (0)
  if (!s->cap_stream) GTRY(cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
  if (!s->cap_stream2) GTRY(cudaStreamCreateWithFlags(&s->cap_stream2, cudaStreamNonBlocking));
  cudaStream_t st = s->cap_stream, st2 = s->cap_stream2;
  cudaStreamCaptureStatus cs;
  cudaGraph_t cg = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t nd = 0;
  int rc;
  const unsigned long long l0 = g_launch_count;
  GTRY(cudaStreamBeginCapture(st, cudaStreamCaptureModeRelaxed));
  // every conditional node owns its handles (default 0 at each graph launch); the kernels enqueued
  // below capture them by value
  cudaGraphConditionalHandle hif[8], hwh[8];
  GTRY(cudaStreamGetCaptureInfo_v2(st, &cs, nullptr, &cg, &deps, &nd));
  for (int copy = 0; copy < copies; ++copy) {
    GTRY(cudaGraphConditionalHandleCreate(&hif[copy], cg, 0, cudaGraphCondAssignDefault));
    GTRY(cudaGraphConditionalHandleCreate(&hwh[copy], cg, 0, cudaGraphCondAssignDefault));
  }
  for (int copy = 0; copy < copies; ++copy) {
  s->h_if = hif[copy]; s->h_while = hwh[copy];
  s->h_if_next = (copy + 1 < copies) ? hif[copy + 1] : 0;
  if (copy == 0) {  // later copies: the gate is set by the previous copy's iter_end
    fresh_gate_kernel<<<1, 32, 0, st>>>(s->S, s->h_if);
    ++g_launch_count;
    GTRY(cudaPeekAtLastError());
  }
  {  // IF node: closure() at the current iterate when lbfgs n_iter == 0
    GTRY(cudaStreamGetCaptureInfo_v2(st, &cs, nullptr, &cg, &deps, &nd));
    cudaGraphNodeParams np = {};
    np.type = cudaGraphNodeTypeConditional;
    np.conditional.handle = s->h_if;
    np.conditional.type = cudaGraphCondTypeIf;
    np.conditional.size = 1;
    cudaGraphNode_t node;
    GTRY(cudaGraphAddNode(&node, cg, deps, nd, &np));
    cudaGraph_t body = np.conditional.phGraph_out[0];
    GTRY(cudaStreamBeginCaptureToGraph(st2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    const unsigned long long a = g_launch_count;
    rc = enqueue_fresh(s, st2);
    s->graph_kernels_fresh = (int)(g_launch_count - a);
    cudaError_t e = cudaStreamEndCapture(st2, nullptr);
    if (rc) return rc;
    GTRY(e);
    GTRY(cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));
  }
  if ((rc = enqueue_direction(s, st))) return rc;
  {  // WHILE node: line-search trials
    GTRY(cudaStreamGetCaptureInfo_v2(st, &cs, nullptr, &cg, &deps, &nd));
    cudaGraphNodeParams np = {};
    np.type = cudaGraphNodeTypeConditional;
    np.conditional.handle = s->h_while;
    np.conditional.type = cudaGraphCondTypeWhile;
    np.conditional.size = 1;
    cudaGraphNode_t node;
    GTRY(cudaGraphAddNode(&node, cg, deps, nd, &np));
    cudaGraph_t body = np.conditional.phGraph_out[0];
    GTRY(cudaStreamBeginCaptureToGraph(st2, body, nullptr, nullptr, 0, cudaStreamCaptureModeRelaxed));
    const unsigned long long a = g_launch_count;
    rc = enqueue_trial(s, st2);
    s->graph_kernels_trial = (int)(g_launch_count - a);
    cudaError_t e = cudaStreamEndCapture(st2, nullptr);
    if (rc) return rc;
    GTRY(e);
    GTRY(cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));
  }
  if ((rc = enqueue_finish(s, st))) return rc;
  }  // copies
  GTRY(cudaStreamEndCapture(st, graph_out));
  GTRY(cudaGraphInstantiate(exec_out, *graph_out, 0));
  s->h_if = s->h_while = s->h_if_next = 0;
  if (copies == 1)  // kernels of one iteration outside the conditional bodies (gate included)
    s->graph_kernels_fixed = (int)(g_launch_count - l0) - s->graph_kernels_trial - s->graph_kernels_fresh;
  g_launch_count = l0;  // capture enqueued nothing; launches are counted per graph launch
  return 0;
#undef GTRY
}

}  // namespace

extern "C" {

int mde_solver_create(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m, const mde_solver_opts_t* opts,
                      void* stream) {
  if (!out || !e || !opts || n < 1 || m < 1) return MDE_E_INVALID;
  if (opts->memory_size < 1 || opts->memory_size > kMaxMemory) return MDE_E_UNSUPPORTED;
  if (opts->constraint == MDE_CONSTRAINT_STANDARDIZED && m > kWideMaxM) return MDE_E_UNSUPPORTED;
  if (opts->constraint < 0 || opts->constraint > MDE_CONSTRAINT_ANCHORED) return MDE_E_INVALID;
  if (opts->max_iter < 1) return MDE_E_INVALID;
  if (opts->mode < 0 || opts->mode > 2) return MDE_E_INVALID;
  if (opts->mode == 1 && opts->world_size > 1) return MDE_E_UNSUPPORTED;  // the NCCL hook is called from the host
  if (n != edges_n(e)) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  mde_solver* s = new (std::nothrow) mde_solver();
  if (!s) return MDE_E_ALLOC;
  s->edges = e; s->n = n; s->m = m; s->N = n * m; s->opts = *opts;
  s->npad = ((s->N + 31) / 32) * 32;
  const int64_t vb = (s->npad + 32) * sizeof(float);  // room for the (hi, lo) tail
  int rc = 0;
#define TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { rc = (int)_e; goto fail; } } while (0)
  TRY(cudaMalloc(&s->S, sizeof(SolverState)));
  TRY(cudaMallocHost(&s->status_host, kStatusInts * sizeof(int)));
  TRY(cudaMalloc(&s->X, vb)); TRY(cudaMalloc(&s->xinit, vb)); TRY(cudaMalloc(&s->d, vb));
  TRY(cudaMalloc(&s->gprev, vb));
  if (opts->world_size > 1) {
    if (opts->world_size > kMaxWorld) { rc = MDE_E_UNSUPPORTED; goto fail; }
    // one peer-visible region: [partial buffer | g (peers store the reduced chunks here) | W receive slots |
    //                           tails | fa[W] fb[W] fd[W] (64 B apart) | epoch | ticket]
    const int64_t vba = (vb + 255) / 256 * 256;
    const int64_t n4 = s->npad >> 2;
    const bool big = (s->npad + 4) * (int64_t)sizeof(float) > kOneShotBytes;
    s->comm_slot_floats = big ? (((n4 + opts->world_size - 1) / opts->world_size) * 4 + 63) / 64 * 64 : 0;
    s->comm_g_off = vba;
    s->comm_recv_off = 2 * vba;
    s->comm_tails_off = s->comm_recv_off + (int64_t)opts->world_size * s->comm_slot_floats * (int64_t)sizeof(float);
    s->comm_flags_off = (s->comm_tails_off + 2 * kMaxWorld * (int64_t)sizeof(float) + 255) / 256 * 256;
    s->comm_bytes = s->comm_flags_off + 64 * (3 * kMaxWorld + 2);
    TRY(cudaMalloc(&s->comm_region, s->comm_bytes));
    TRY(cudaMemsetAsync(s->comm_region, 0, s->comm_bytes, st));
    TRY(cudaMalloc(&s->comm_dev, sizeof(Comm)));
    s->gpart = reinterpret_cast<float*>(s->comm_region);
    s->g = reinterpret_cast<float*>(reinterpret_cast<char*>(s->comm_region) + s->comm_g_off);
    { const char* ev = getenv("MDE_B200_ALLREDUCE"); if (ev && !strcmp(ev, "pull")) s->comm_pull = 1; }
  } else {
    TRY(cudaMalloc(&s->g, vb));
  }
  TRY(cudaMalloc(&s->Sb, (int64_t)(opts->memory_size + 1) * s->npad * sizeof(float)));
  TRY(cudaMalloc(&s->Yb, (int64_t)(opts->memory_size + 1) * s->npad * sizeof(float)));
  TRY(cudaMalloc(&s->dpart, sizeof(double) * (int64_t)kVecBlocks * kHeadCols * kMaxSlices));
  TRY(cudaMalloc(&s->vpart, sizeof(double) * (int64_t)kVecBlocks * 4));
  TRY(cudaMemsetAsync(s->vpart, 0, sizeof(double) * (int64_t)kVecBlocks * 4, st));
  TRY(cudaMalloc(&s->stats, sizeof(double) * 4 * (int64_t)opts->max_iter));
  TRY(cudaMalloc(&s->projws, mde_project_ws_bytes(n, m)));
  s->pw = proj_ws_carve(s->projws, m);
  TRY(cudaMemsetAsync(s->X, 0, vb, st)); TRY(cudaMemsetAsync(s->xinit, 0, vb, st));
  TRY(cudaMemsetAsync(s->d, 0, vb, st)); TRY(cudaMemsetAsync(s->g, 0, vb, st));
  TRY(cudaMemsetAsync(s->gprev, 0, vb, st));
  TRY(cudaMemsetAsync(s->Sb, 0, (int64_t)(opts->memory_size + 1) * s->npad * sizeof(float), st));
  TRY(cudaMemsetAsync(s->Yb, 0, (int64_t)(opts->memory_size + 1) * s->npad * sizeof(float), st));
  if (opts->constraint == MDE_CONSTRAINT_ANCHORED && opts->n_anchors > 0) {
    if (!opts->anchors || !opts->anchor_values) { rc = MDE_E_INVALID; goto fail; }
    TRY(cudaMalloc(&s->anchors, sizeof(int64_t) * opts->n_anchors));
    TRY(cudaMalloc(&s->anchor_values, sizeof(float) * opts->n_anchors * m));
    TRY(cudaMemcpyAsync(s->anchors, opts->anchors, sizeof(int64_t) * opts->n_anchors, cudaMemcpyDeviceToDevice, st));
    TRY(cudaMemcpyAsync(s->anchor_values, opts->anchor_values, sizeof(float) * opts->n_anchors * m,
                        cudaMemcpyDeviceToDevice, st));
  }
  s->nvb = vec_blocks(s->npad >> 2);
  if (opts->constraint == MDE_CONSTRAINT_CENTERED && (m == 1 || m == 2 || m == 4)) s->center_m = m;
  { const char* ev = getenv("MDE_B200_FUSE"); if (ev && ev[0] == '0') s->fuse = 0; }
  if (opts->mode == 2) {
    s->fuse = 1;  // the phase machine lives in the fused epilogues
    s->late = 1;
    const char* ev = getenv("MDE_B200_LATE");
    if (ev && ev[0] == '0') s->late = 0;
  }
  if (opts->mode == 2 && opts->world_size == 1) {  // several GPUs: graphs are built by mde_solver_comm_connect
    s->nl = 0;
    TRY(cudaStreamSynchronize(st));
    rc = build_step_graph(s, 1, &s->step_graph, &s->step_exec);
    if (rc) goto fail;
    { const char* ev = getenv("MDE_B200_STEPS"); if (ev) s->steps_per_graph = atoi(ev); }
    if (s->steps_per_graph < 1) s->steps_per_graph = 1;
    if (s->steps_per_graph > 64) s->steps_per_graph = 64;
    rc = build_step_graph(s, s->steps_per_graph, &s->steps_graph, &s->steps_exec);
    if (rc) goto fail;
  }
  if (opts->mode == 1) {
    s->nl = 0;
    TRY(cudaStreamSynchronize(st));
    rc = build_iteration_graph(s, 1, &s->graph, &s->graph_exec);
    if (rc) goto fail;
    { const char* ev = getenv("MDE_B200_UNROLL"); if (ev) s->unroll = atoi(ev); }
    if (s->unroll < 1) s->unroll = 1;
    if (s->unroll > 8) s->unroll = 8;
    if (s->unroll > 1) {
      rc = build_iteration_graph(s, s->unroll, &s->graph_u, &s->graph_exec_u);
      if (rc) goto fail;
    }
  }
  *out = s;
  return 0;
fail:
  mde_solver_destroy(s);
  return rc;
#undef TRY
}

int mde_solver_destroy(mde_solver_t* s) {
  if (!s) return 0;
  cudaFree(s->S); cudaFreeHost(s->status_host);
  cudaFree(s->X); cudaFree(s->xinit); cudaFree(s->d); cudaFree(s->gprev);
  if (!s->comm_region) cudaFree(s->g);  // (several GPUs: g lives inside the peer-visible region)
  for (int q = 0; q < kMaxWorld; ++q) if (s->peer_base[q]) cudaIpcCloseMemHandle(s->peer_base[q]);
  cudaFree(s->comm_region); cudaFree(s->comm_dev);
  cudaFree(s->Sb); cudaFree(s->Yb); cudaFree(s->dpart); cudaFree(s->vpart); cudaFree(s->stats); cudaFree(s->projws);
  cudaFree(s->anchors); cudaFree(s->anchor_values);
  if (s->graph_exec) cudaGraphExecDestroy(s->graph_exec);
  if (s->graph) cudaGraphDestroy(s->graph);
  if (s->step_exec) cudaGraphExecDestroy(s->step_exec);
  if (s->step_graph) cudaGraphDestroy(s->step_graph);
  if (s->steps_exec) cudaGraphExecDestroy(s->steps_exec);
  if (s->steps_graph) cudaGraphDestroy(s->steps_graph);
  if (s->graph_exec_u) cudaGraphExecDestroy(s->graph_exec_u);
  if (s->graph_u) cudaGraphDestroy(s->graph_u);
  if (s->cap_stream) cudaStreamDestroy(s->cap_stream);
  if (s->cap_stream2) cudaStreamDestroy(s->cap_stream2);
  delete s;
  return 0;
}

int mde_solver_set_allreduce(mde_solver_t* s, mde_allreduce_fn fn, void* user) {
  if (!s) return MDE_E_INVALID;
  s->allreduce = fn; s->allreduce_user = user;
  return 0;
}

int mde_solver_comm_export(mde_solver_t* s, void* handle_out, int64_t handle_bytes) {
  if (!s || !handle_out || !s->comm_region || handle_bytes < (int64_t)sizeof(cudaIpcMemHandle_t)) return MDE_E_INVALID;
  cudaIpcMemHandle_t h;
  MDE_CUDA_TRY(cudaIpcGetMemHandle(&h, s->comm_region));
  memcpy(handle_out, &h, sizeof(h));
  return 0;
}

int mde_solver_comm_connect(mde_solver_t* s, int rank, const void* handles, int64_t handle_stride, void* stream) {
  if (!s || !handles || !s->comm_region || rank < 0 || rank >= s->opts.world_size ||
      handle_stride < (int64_t)sizeof(cudaIpcMemHandle_t))
    return MDE_E_INVALID;
  if (s->comm_connected) return MDE_E_INVALID;
  if (s->opts.mode != 2) return MDE_E_UNSUPPORTED;  // host-stepped modes keep the host hook
  cudaStream_t st = (cudaStream_t)stream;
  const int W = s->opts.world_size;
  Comm c{};
  c.rank = rank; c.world = W;
  for (int q = 0; q < W; ++q) {
    char* base;
    if (q == rank) base = reinterpret_cast<char*>(s->comm_region);
    else {
      cudaIpcMemHandle_t h;
      memcpy(&h, reinterpret_cast<const char*>(handles) + (int64_t)q * handle_stride, sizeof(h));
      void* ptr = nullptr;
      MDE_CUDA_TRY(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
      s->peer_base[q] = ptr;
      base = reinterpret_cast<char*>(ptr);
    }
    char* fl = base + s->comm_flags_off;
    c.buf[q] = reinterpret_cast<float*>(base);
    c.fa[q] = reinterpret_cast<unsigned*>(fl);
    c.fb[q] = reinterpret_cast<unsigned*>(fl + 64 * kMaxWorld);
    c.fd[q] = reinterpret_cast<unsigned*>(fl + 64 * 2 * kMaxWorld);
    c.gout[q] = reinterpret_cast<float*>(base + s->comm_g_off);
    c.recv[q] = reinterpret_cast<float*>(base + s->comm_recv_off);
    c.tails[q] = reinterpret_cast<float*>(base + s->comm_tails_off);
  }
  c.slot_floats = s->comm_slot_floats;
  {
    char* fl = reinterpret_cast<char*>(s->comm_region) + s->comm_flags_off;
    c.epoch = reinterpret_cast<unsigned*>(fl + 64 * 3 * kMaxWorld);
    c.ticket = reinterpret_cast<unsigned*>(fl + 64 * (3 * kMaxWorld + 1));
  }
  s->comm = c;
  MDE_CUDA_TRY(cudaMemcpyAsync(s->comm_dev, &s->comm, sizeof(Comm), cudaMemcpyHostToDevice, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  s->comm_connected = 1;
  if (s->opts.mode == 2) {  // the sharded solve runs the same flat step graphs as one GPU
    s->nl = 0;
    int rc = build_step_graph(s, 1, &s->step_graph, &s->step_exec);
    if (rc) return rc;
    { const char* ev = getenv("MDE_B200_STEPS"); if (ev) s->steps_per_graph = atoi(ev); }
    if (s->steps_per_graph < 1) s->steps_per_graph = 1;
    if (s->steps_per_graph > 64) s->steps_per_graph = 64;
    rc = build_step_graph(s, s->steps_per_graph, &s->steps_graph, &s->steps_exec);
    if (rc) return rc;
  }
  return 0;
}

int mde_solver_begin(mde_solver_t* s, const float* X0, double eps, void* stream) {
  return mde_solver_begin_ex(s, X0, eps, s ? s->opts.max_iter : 0, stream);
}

int mde_solver_begin_ex(mde_solver_t* s, const float* X0, double eps, int max_iter, void* stream) {
  if (!s || !X0) return MDE_E_INVALID;
  if (max_iter < 1 || max_iter > s->opts.max_iter) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  MDE_CUDA_TRY(cudaMemcpyAsync(s->X, X0, sizeof(float) * s->N, cudaMemcpyDeviceToDevice, st));
  const int mi = s->opts.max_iter;  // stride of the statistics arrays (capacity)
  s->cur_max_iter = max_iter;
  init_state_kernel<<<1, 32, 0, st>>>(s->S, eps, s->opts.memory_size, max_iter, s->opts.world_size, s->stats,
                                      s->stats + mi, s->stats + 2 * mi, s->stats + 3 * mi);
  MDE_LAUNCH_CHECK();
  s->host_need_fresh = 1;
  s->host_active = 1;
  s->host_evals = 0;
  s->host_iter = 0;
  return 0;
}

// globaltimer stamps (ns) of the last late-epilogue head kernel that started an iteration: [0] last block's entry,
// [1] epilogue entry, [2] state staged, [3] partials reduced, [4] previous step finished, [5] direction done,
// [6] before write-back, [7] the vec kernel's first block.  Diagnostics only (tools/solver_times.py).
int mde_solver_debug_times(mde_solver_t* s, unsigned long long* out8, void* stream) {
  if (!s || !out8) return MDE_E_INVALID;
  MDE_CUDA_TRY(cudaMemcpyAsync(out8, s->S->dbg, sizeof(unsigned long long) * 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  MDE_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

int mde_solver_run(mde_solver_t* s, int iters, int* iters_done, int* converged, void* stream) {
  if (!s) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = 0;
  if (s->opts.mode == 2) {
    // flat step graphs: the device pauses itself at `target`; the host only keeps the queue fed.  A step is
    // one closure evaluation, an iteration takes >= 1 of them, so launching `remaining` steps never overshoots
    // by more than the gated (early-exit) kernels of the surplus steps.
    if (!s->host_active || iters <= 0) {
      if ((rc = read_status(s, st))) return rc;
      if (iters_done) *iters_done = s->status_host[2];
      if (converged) *converged = s->status_host[1];
      return 0;
    }
    int target = s->host_iter + iters;
    if (target > s->cur_max_iter) target = s->cur_max_iter;
    resume_kernel<<<1, 32, 0, st>>>(s->S, target);
    MDE_LAUNCH_CHECK();
    for (int round = 0;; ++round) {
      if (round > (1 << 18)) return MDE_E_INVALID;
      int remaining = target - s->host_iter;
      if (remaining < 1) remaining = 1;
      long long steps = 0;
      const int spg = s->steps_per_graph;
      if (s->opts.world_size > 1 && !s->steps_exec) {
        // host-hook all-reduce: stream-launched steps; every rank enqueues the same number of steps (same `remaining`: the replicated state machines agree)
        int n_steps = remaining + remaining / 8 + (round > 0 ? 1 : 0) + s->late;
        if (n_steps > 64) n_steps = 64;
        for (int b = 0; b < n_steps; ++b) { if ((rc = enqueue_step(s, st))) return rc; }
      } else if (remaining >= spg) {
        int graphs = (remaining + remaining / 8 + s->late) / spg;
        if (graphs * spg > 96) graphs = 96 / spg > 0 ? 96 / spg : 1;  // <= ~96 steps in flight per status read
        for (int b = 0; b < graphs; ++b) MDE_CUDA_TRY(cudaGraphLaunch(s->steps_exec, st));
        steps = (long long)graphs * spg;
      } else {
        const int singles = remaining + remaining / 4 + (round > 0 ? 1 : 0) + s->late;
        for (int b = 0; b < singles; ++b) MDE_CUDA_TRY(cudaGraphLaunch(s->step_exec, st));
        steps = singles;
      }
      g_launch_count += (unsigned long long)steps * s->step_kernels;  // (stream-launched steps count themselves)
      if ((rc = read_status(s, st))) return rc;
      s->host_iter = s->status_host[2];
      if (s->status_host[3]) { s->host_active = 0; if (iters_done) *iters_done = s->status_host[2]; return s->status_host[3]; }
      if (!s->status_host[0]) {              // paused at the target, converged, or out of iterations
        s->host_active = s->status_host[8];  // only a pause can be resumed
        break;
      }
    }
    if (iters_done) *iters_done = s->status_host[2];
    if (converged) *converged = s->status_host[1];
    return 0;
  }
  if (s->opts.mode == 1) {
    // device-driven: one graph launch per iteration, status read back once per batch.  Launches
    // after convergence are no-ops (every kernel checks the device-side `active` flag).
    int left = iters;
    while (left > 0 && s->host_active) {
      const int batch = left < 16 ? left : 16;
      int b = 0, chained = 0;
      for (; s->unroll > 1 && b + s->unroll <= batch; b += s->unroll, ++chained)
        MDE_CUDA_TRY(cudaGraphLaunch(s->graph_exec_u, st));
      for (; b < batch; ++b) MDE_CUDA_TRY(cudaGraphLaunch(s->graph_exec, st));
      left -= batch;
      if ((rc = read_status(s, st))) return rc;
      s->host_active = s->status_host[0];
      // kernels executed by the graphs: fixed part per launch + one trial body per evaluation
      g_launch_count += (unsigned long long)batch * s->graph_kernels_fixed +
                        (unsigned long long)(s->status_host[7] - s->host_evals) * s->graph_kernels_trial;
      g_launch_count -= (unsigned long long)chained * (s->unroll - 1);  // chained copies carry no gate kernel
      s->host_evals = s->status_host[7];
      if (s->status_host[3]) { if (iters_done) *iters_done = s->status_host[2]; return s->status_host[3]; }
    }
    if ((rc = read_status(s, st))) return rc;
    if (iters_done) *iters_done = s->status_host[2];
    if (converged) *converged = s->status_host[1];
    return 0;
  }
  for (int it = 0; it < iters && s->host_active; ++it) {
    if (s->host_need_fresh) { if ((rc = enqueue_fresh(s, st))) return rc; }
    if ((rc = enqueue_direction(s, st))) return rc;
    for (int trial = 0;; ++trial) {  // <= 10 back-offs + 25 search steps + ~85 fallback steps
      if (trial > 256) return MDE_E_INVALID;
      if ((rc = enqueue_trial(s, st))) return rc;
      if ((rc = read_status(s, st))) return rc;
      if (!s->status_host[5] || !s->status_host[0]) break;  // ls_active / active
    }
    if (s->status_host[3]) { s->host_active = 0; if (iters_done) *iters_done = s->status_host[2]; return s->status_host[3]; }
    if ((rc = enqueue_finish(s, st))) return rc;
    if ((rc = read_status(s, st))) return rc;
    s->host_need_fresh = s->status_host[4];
    s->host_active = s->status_host[0];
  }
  if ((rc = read_status(s, st))) return rc;
  if (iters_done) *iters_done = s->status_host[2];
  if (converged) *converged = s->status_host[1];
  return 0;
}

float* mde_solver_x(mde_solver_t* s) { return s ? s->X : nullptr; }

int mde_solver_stats(mde_solver_t* s, double* avg, double* resid, double* pct, double* steplen,
                     int64_t* func_evals, void* stream) {
  if (!s) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = read_status(s, st);
  if (rc) return rc;
  const int it = s->status_host[2];
  const int mi = s->opts.max_iter;
  if (avg) MDE_CUDA_TRY(cudaMemcpyAsync(avg, s->stats, sizeof(double) * it, cudaMemcpyDeviceToHost, st));
  if (resid) MDE_CUDA_TRY(cudaMemcpyAsync(resid, s->stats + mi, sizeof(double) * it, cudaMemcpyDeviceToHost, st));
  if (pct) MDE_CUDA_TRY(cudaMemcpyAsync(pct, s->stats + 2 * mi, sizeof(double) * it, cudaMemcpyDeviceToHost, st));
  if (steplen) MDE_CUDA_TRY(cudaMemcpyAsync(steplen, s->stats + 3 * mi, sizeof(double) * it, cudaMemcpyDeviceToHost, st));
  if (func_evals) {
    long long fe = 0;
    MDE_CUDA_TRY(cudaMemcpyAsync(&fe, (const char*)s->S + offsetof(SolverState, func_evals), sizeof(long long),
                                 cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaStreamSynchronize(st));
    *func_evals = fe;
  }
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// ---- host-side debug entry points: the scalar logic above, runnable without a GPU ----------
void* mde_dbg_ls_new(double t0, double f0, float gtd0, float d_norm) {
  LsState* L = new LsState();
  ls_begin(*L, t0, f0, gtd0, d_norm);
  return L;
}
void mde_dbg_ls_free(void* p) { delete (LsState*)p; }
double mde_dbg_ls_t(void* p) { return ((LsState*)p)->t; }
int mde_dbg_ls_step(void* p, double f_new, float gtd_new, int grad_finite) {
  LsState* L = (LsState*)p;
  ls_on_result(*L, f_new, gtd_new, grad_finite != 0);
  return L->phase;
}
void mde_dbg_ls_result(void* p, double* t_accept, double* f_accept, int* func_evals, int* error) {
  LsState* L = (LsState*)p;
  *t_accept = L->t_accept; *f_accept = L->f_accept; *func_evals = L->func_evals; *error = L->error;
}
void* mde_dbg_lbfgs_new(int memory) {
  LbfgsState* B = new LbfgsState();
  lbfgs_reset(*B, memory);
  return B;
}
void mde_dbg_lbfgs_free(void* p) { delete (LbfgsState*)p; }
// one direction update; arrays have kMaxMemory+1 entries.  Outputs: count, cand, order, coefficients.
void mde_dbg_lbfgs_step(void* p, double ys, double yy, double sc_g, double yc_g, double* sj_yc, double* yj_yc,
                        double* sc_yj, double* sj_g, double* yj_g, int* count, int* cand, int* order, double* cg,
                        double* cs, double* cy) {
  LbfgsState* B = (LbfgsState*)p;
  lbfgs_direction(*B, B->SY, B->YY, ys, yy, sc_g, yc_g, sj_yc, yj_yc, sc_yj, sj_g, yj_g);
  *count = B->count; *cand = B->cand; *cg = B->cg;
  for (int j = 0; j < B->count; ++j) { order[j] = B->order[j]; cs[j] = B->cs[j]; cy[j] = B->cy[j]; }
}
void mde_dbg_lbfgs_reset(void* p) { LbfgsState* B = (LbfgsState*)p; lbfgs_reset(*B, B->memory); }
int mde_dbg_lbfgs_cand(void* p) { return ((LbfgsState*)p)->cand; }

}  // extern "C"
