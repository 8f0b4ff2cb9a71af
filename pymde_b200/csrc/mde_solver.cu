// mde_solver.cu -- device-resident projected L-BFGS (the MDE.embed solve loop).
//
// Replaces optim.lbfgs (pymde/optim.py:69-184) driving LBFGS.step (pymde/lbfgs.py:390-590),
// _strong_wolfe (pymde/lbfgs.py:44-253), the value_and_grad closure (pymde/optim.py:100-105)
// and the per-iteration callback/statistics (pymde/optim.py:94-96,139-173).
//
// Design:
//  * every vector (X, x_init, d, g, g_prev, the S/Y history ring) and every scalar (loss,
//    g.d, Wolfe bracket, Gram matrix of the history, statistics) lives in HBM; the host
//    only launches CUDA graphs of identical "steps" (one closure evaluation each, every kernel
//    gated by a device-side phase machine) and reads one 48-byte status word per batch of steps;
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
#include <chrono>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <new>

#include "mde_edges.cuh"
#include "mde_logic.h"
#include "mde_project.cuh"

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
constexpr int kStepsPerGraph = 8;  // steps of the multi-step graph (the one-step graph takes the last few)
enum { PH_DIR = 0, PH_TRIAL = 1, PH_FRESH = 2, PH_MAT = 3 };  // phase of a step

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
  // ---- step phase machine ----
  int paused;      // stopped at iter_limit; mde_solver_run resumes it
  int phase;       // what the next step does (PH_*)
  int iter_limit;  // pause when `iter` reaches it
  int pend;        // 1 = the previous step executed phase `phase`, its bookkeeping is pending
  int g_eval;      // gates of the next step, written by the head kernel's epilogue: closure evaluation runs
  int g_proj;      //   the iterate moved: retraction kernels run
  unsigned int ticket;  // last-block-done counter of the head kernel
  int run_seq;     // of the mde_solver_run call that armed the solver (progress word)
  int run_steps;   // head kernels that ran their scalar stage since that call armed it
  // ---- scalars ----
  double eps;
  double loss;     // f at the current iterate (cached loss, lbfgs.py:418-426,550)
  double gg, g1;   // ||g||^2 and ||g||_1 of the gradient buffer
  double dd, xx;   // ||d||^2, ||X||^2 at iteration start
  float mu_x[4], mu_d[4];  // column means of x_init and d (Centered, m in {1,2,4}: fused into the vec kernel)
  double t_last;   // state["t"]
  double t_eval;   // step of the most recent trial evaluation
  long long func_evals;
  int max_stats;
  int world;
  double *avg, *resid, *pct, *steplen;
  double t_cur;                      // step length the current step's vec kernel applies (t0 / ls.t / ls.t_accept)
  double cs_g[4], cs_d[4];           // column sums of g_prev and d (tracked through the two-loop coefficients)
  double cs_S[kSlots][4], cs_Y[kSlots][4];  // ... and of the stored pairs
  HeadDesc hd;                       // written by init / the head kernel's epilogue for the NEXT head kernel
  unsigned long long dbg[12];        // globaltimer stamps of the last head kernel that started an iteration (mde_solver_debug_times)
  LsState ls;
  LbfgsState lb;
};

__device__ __forceinline__ bool off(const int* flag) { return *flag == 0; }

// Progress word: one 64-bit word in mapped host memory that resume_kernel and every head kernel's scalar stage
// overwrite, so that mde_solver_run can keep the step queue fed, and see the solve stop, without synchronising.  One
// 8-byte store is single-copy atomic, so the host always reads one consistent snapshot and the store needs no fence.
// Layout: [63] stopped (not active), [62] paused, [61] converged, [60] failed, [59:53] run sequence number,
// [52:32] steps of this run modulo 2^21, [31:0] completed iterations.
constexpr int kProgSeqMask = 0x7f;
constexpr long long kProgStepsMask = (1ll << 21) - 1;

__device__ __forceinline__ void publish_progress(unsigned long long* p, const SolverState* S) {
  const unsigned long long w =
      ((unsigned long long)(S->active ? 0 : 1) << 63) | ((unsigned long long)(S->paused ? 1 : 0) << 62) |
      ((unsigned long long)(S->converged ? 1 : 0) << 61) | ((unsigned long long)(S->error ? 1 : 0) << 60) |
      ((unsigned long long)(S->run_seq & kProgSeqMask) << 53) | ((unsigned long long)(S->run_steps & kProgStepsMask) << 32) |
      (unsigned long long)(unsigned)S->iter;
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(w) : "memory");
}

struct Progress {
  bool stopped, paused, converged, failed;
  int seq, iter;
  long long steps;
};

inline Progress decode_progress(unsigned long long w) {
  return {(w >> 63 & 1) != 0, (w >> 62 & 1) != 0, (w >> 61 & 1) != 0, (w >> 60 & 1) != 0,
          (int)(w >> 53 & kProgSeqMask), (int)(unsigned)w, (long long)(w >> 32 & kProgStepsMask)};
}

// Fixed-order reduction of K sums over nb block partials into smem out[K]; all threads of the block call.
// Stage 1: thread t owns (k = t % K, segment = t / K) and walks blocks segment, segment + S, ... in batches of
// 16 independent coalesced loads (through L2: the partials may come from other SMs of the same launch).
// Stage 2: one warp per output combines the S segment sums with a fixed shuffle tree.  The summation order
// depends only on (nb, K, blockDim), so scalars are bit-reproducible for a given launch shape.
__device__ void reduce_partials(const double* __restrict__ part, int nb, int K, double* out) {
  __shared__ double red_buf[256];
  const int T = blockDim.x < 256 ? blockDim.x : 256;
  const int S = T / K;  // segments (K < T)
  const int k = threadIdx.x % K, seg = threadIdx.x / K;
  if (threadIdx.x < S * K) {
    constexpr int U = 16;
    double s = 0.0;
    for (int b0 = seg; b0 < nb; b0 += U * S) {
      double v[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int b = b0 + u * S;
        v[u] = (b < nb) ? __ldcg(part + (int64_t)b * K + k) : 0.0;
      }
#pragma unroll
      for (int u = 0; u < U; ++u) s += v[u];
    }
    red_buf[seg * K + k] = s;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (int)(blockDim.x >> 5);
  for (int kk = w; kk < K; kk += nw) {  // warp-uniform trip count
    double s = 0.0;
    for (int q = lane; q < S; q += 32) s += red_buf[q * K + kk];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(kFull, s, o);
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

struct Tail {              // what the head kernel's scalar epilogue needs
  const double* lpart;     // loss partials of the distortion launch
  int nl;
  const float* tail;       // (hi, lo) of the all-reduced loss (multi-GPU)
  double p_total;
  double inv_n;            // 1 / n_rows
};

// ---------------------------------------------------------------------------------------
// history update + two-loop in Gram form
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

// anchored constraint (pymde/constraints.py:114-164): overwrite / zero anchor rows
__global__ void anchor_rows_kernel(const int* flag, float* __restrict__ Z, const int64_t* __restrict__ anchors,
                                   const float* __restrict__ values, int64_t na, int m) {
  if (off(flag)) return;
  int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= na * m) return;
  int64_t a = anchors[i / m];
  Z[a * m + (i % m)] = values ? values[i] : 0.0f;
}

// multi-GPU: the all-reduced [gradient | loss] becomes the solver's gradient buffer -- only when the
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
  reduce_partials(lpart, nl, 1, out);
  if (threadIdx.x == 0) {
    float hi = (float)out[0];
    tail[0] = hi;
    tail[1] = (float)(out[0] - (double)hi);
  }
}

// callable distortion function: the coefficients g_k = f'(d_k) / d_k the scatter takes (the caller's torch code left
// fpp = d mean f / d d), non-finite g replaced by 1 like the reference (pymde/average_distortion.py:55-62), and the loss
// sum f(d).sum() in the layout's first loss-partial slot, where the next head kernel reads it (one partial)
__global__ void __launch_bounds__(256)
ext_coeff_kernel(const int* flag, const float* __restrict__ fpp, const float* __restrict__ d,
                 const double* __restrict__ loss, float* __restrict__ g, double* __restrict__ lpart, int64_t p) {
  if (off(flag)) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < p; k += stride) {
    const float v = __fdiv_rn(fpp[k], d[k]);  // IEEE division: the same floats as the torch path
    g[k] = isfinite(v) ? v : 1.0f;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) lpart[0] = *loss;
}

// ---------------------------------------------------------------------------------------
// Multi-GPU (SURVEY section 8e): edge shards, X replicated, ONE all-reduce of [gradient | loss] per evaluation.
// The all-reduce is done by OUR kernels over NVLink peer memory (cudaIpc-mapped buffers of the other ranks), not by
// a host-side NCCL call: plain kernel nodes, so the sharded solve runs the same CUDA graph of gated steps as one
// GPU, and a gated-off step costs nothing.  Every rank sums the peers' partial buffers in RANK ORDER, so all ranks
// hold bit-identical gradients (the replicated Wolfe / L-BFGS decisions depend on it).
//   small buffers (<= kOneShotBytes): one-shot -- every rank reads all W partial buffers and writes g
//   (allreduce_kernel);
//   large buffers: write-based -- rank r stores chunk q of its partial buffer into rank q's receive slots, rank q
//   sums its W copies and stores the reduced chunk into the gradient buffer of every rank (allreduce_push_kernel):
//   every byte crosses NVLink as a posted store.
// Handshake: monotonically increasing epochs in per-rank flag arrays (st.release.sys / ld.acquire.sys),
// fa = "my partial buffer is complete" (one-shot) / "my chunks are in the peers' receive slots" (write-based),
// fb = "my reduced chunk is in every rank's g", fd = "I have finished reading the peers".
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

// One-shot: g[i] = sum_q buf_q[i] (rank order) for i < npad, tail summed in double.
__global__ void __launch_bounds__(kCommThreads)
allreduce_kernel(const int* __restrict__ flag, Comm c, float* __restrict__ g, int64_t npad, int* __restrict__ err) {
  if (off(flag)) return;
  const unsigned ep = *reinterpret_cast<volatile unsigned*>(c.epoch) + 1u;
  if (blockIdx.x == 0) comm_signal(c.fa, c, ep);
  comm_wait(c.fa[c.rank], c, ep, err);
  const int64_t n4 = npad >> 2;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  constexpr int U = 2;  // float4 per thread per trip; all U * world peer loads are issued before the first add
  for (int64_t i0 = tid; i0 < n4; i0 += U * stride) {
    float4 v[kMaxWorld][U];
#pragma unroll
    for (int q = 0; q < kMaxWorld; ++q) {
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int64_t i = i0 + u * stride;
        v[q][u] = (q < c.world && i < n4) ? ld_peer_f4(c.buf[q] + 4 * i) : make_float4(0.f, 0.f, 0.f, 0.f);
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
      if (i < n4) reinterpret_cast<float4*>(g)[i] = acc;
    }
  }
  if (tid == 0) comm_reduce_tail(c, npad, g + npad);
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

// ---------------------------------------------------------------------------------------
// Large buffers: write-based ("push") all-reduce.  NVLink stores are posted, loads are round trips: a read-based
// reduce-scatter + all-gather sustained ~300 GB/s per GPU on 80 MB gradients.  Here every byte crosses NVLink as a
// store:
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

// end of iteration (optim.py:135-173)
__device__ void iter_end_body(SolverState* __restrict__ S) {
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
}

// ---------------------------------------------------------------------------------------
// The solve as a flat chain of identical "steps" (no conditional graph nodes: an IF or WHILE node costs several
// times a dependent kernel node, tools/microbench/graph_overheads.cu measures them).  A step is
//     head -> vec -> [retraction kernels] -> scatter [-> all-reduce] [-> tangent projection]
// and performs exactly one closure evaluation, with ONE scalar stage, in the head kernel's last block:
//   head  reads g, g_prev, d, X and the history once: (g.d, g.g, |g|_1) of the evaluation the previous step left
//         pending, the history dots of the iteration that would start if that trial is accepted, column sums of g and
//         X (Centered).  Its blocks also fold the previous scatter launch's loss partials and the previous vec
//         kernel's (g.d, d.d, X.X, max|d|) partials into their rows, so the epilogue does one reduction.  Epilogue:
//         finish the previous step (line-search init if it was PH_DIR, Wolfe update, end of iteration), choose this
//         step's phase, and when an iteration starts: history update, two-loop, first step length, column means.
//   vec   PH_DIR: d = H g, g_prev = g, x_init = X and the first trial X = x_init + t0 d in ONE pass (t0 does not
//         depend on g.d: lbfgs.py:521-530); PH_TRIAL / PH_MAT: X = x_init + t d; every phase but PH_MAT: g = 0.
// The epilogue advances a small phase machine and writes the gates the next step's kernels read:
//   PH_FRESH  closure at the current iterate (lbfgs n_iter == 0)           -> PH_DIR
//   PH_DIR    new direction + first line-search trial                      -> PH_TRIAL | PH_MAT | end of iteration
//   PH_TRIAL  another trial of the same line search                        -> PH_TRIAL | PH_MAT | end of iteration
//   PH_MAT    X = retract(x_init + t_accept d) when the accepted step is not the last one evaluated
//             (otherwise X already holds it bit for bit); no evaluation     -> end of iteration
// End of iteration (iter_end_body) -> PH_DIR, or PH_FRESH after a reset, or pause at iter_limit.
// The history dots are SPECULATIVE (they assume the trial just evaluated, t = t_cur, is accepted, which the
// strong-Wolfe search does ~9 times out of 10); when it asks for another trial they are unused, when it accepts an
// earlier point (PH_MAT) the step after the materialisation recomputes them with the accepted t.
// ---------------------------------------------------------------------------------------
__device__ void set_phase(SolverState* __restrict__ S, int ph) {
  S->phase = ph;
  S->need_fresh = (ph == PH_FRESH) ? 1 : 0;
  const int on = S->active;
  S->g_eval = (on && ph != PH_MAT) ? 1 : 0;
  S->g_proj = (on && ph != PH_FRESH) ? 1 : 0;
}

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

// The scalar stage of a step (last block of the head kernel).  The whole SolverState (history Gram
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
                               unsigned char* smem, float tpass, int count, unsigned long long t_entry,
                               unsigned long long* progress) {
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
          sS->dd = sums[kColVec + 1]; sS->xx = sums[kColVec + 2];
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
        iter_end_body(sS);
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
    sS->run_steps += 1;
    publish_progress(progress, sS);
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
                 const double* __restrict__ vpart, Tail tl, unsigned long long* progress) {
  if (off(&S->active)) return;
  __shared__ __align__(16) unsigned char raw[(kHeadSmemBytes + 15) / 16 * 16];  // warp sums, then the scalar stage
  static_assert(sizeof(raw) >= sizeof(float) * kHeadAcc * (kVecThreads / 32), "warp sums must fit");
  static_assert(kHeadAcc == 66, "the transposing butterfly below is written for 64 + 2 accumulators");
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
    int nval = want_hist ? count - slice * kPairsPerSlice : 0;
    if (nval > kPairsPerSlice) nval = kPairsPerSlice;
    // Physical slots of the slice's pairs: lane L of warp 0 picks order byte L of the descriptor with selects (no
    // local array), one shuffle hands pair j's byte to lane j.  The pairs are read through the read-only path
    // (LDG.CONSTANT, addresses formed from Sb / Yb, not pointers kept in shared memory) although Sb / Yb are written
    // in this launch: slice 0 only writes the candidate slot h1.x (lb.cand), which lbfgs_update never leaves in
    // order[0 .. count-1].
    __shared__ int q[kPairsPerSlice];
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      const uint4 hw = (lane < 16) ? h2 : h3;
      const int wi = (lane >> 2) & 3;
      const unsigned word = wi == 0 ? hw.x : (wi == 1 ? hw.y : (wi == 2 ? hw.z : hw.w));
      const int obyte = (int)((word >> (8 * (lane & 3))) & 0xffu);
      const int lj = slice * kPairsPerSlice + lane;
      const int qq = __shfl_sync(kFull, obyte, lj & 31);
      if (lane < kPairsPerSlice) q[lane] = (lj < count) ? qq : 0;
    }
    __syncthreads();
    const int64_t n4 = npad >> 2;
    const int64_t stride = (int64_t)gridDim.x * blockDim.x;
    const float4* S4 = reinterpret_cast<const float4*>(Sb);
    const float4* Y4 = reinterpret_cast<const float4*>(Yb);
    const float4 z4 = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    const bool gh = want_grad || want_hist;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) {
      const float4 G = reinterpret_cast<const float4*>(g)[i];
      const float4 Xv = (slice == 0) ? reinterpret_cast<const float4*>(X)[i] : z4;
      const float4 P = gh ? reinterpret_cast<const float4*>(gprev)[i] : z4;
      const float4 D = gh ? reinterpret_cast<const float4*>(d)[i] : z4;
      const float gv[4] = {G.x, G.y, G.z, G.w};
      if (slice == 0) {
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
      const float dv[4] = {D.x, D.y, D.z, D.w};
      const float yv[4] = {G.x - P.x, G.y - P.y, G.z - P.z, G.w - P.w};
      const float sv[4] = {D.x * t, D.y * t, D.z * t, D.w * t};
      // Every update is computed and then kept or dropped, not branched over (the branchy form spilled at 128
      // registers).  Each accumulator keeps its FFMA chain, so the bits are the same.
      {
        float r0 = acc[kDotsPerSlice], r1 = acc[kDotsPerSlice + 1], r2 = acc[kDotsPerSlice + 2];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          r0 += gv[e] * dv[e];
          r1 += gv[e] * gv[e];
          r2 += fabsf(gv[e]);
        }
        if (want_grad) { acc[kDotsPerSlice] = r0; acc[kDotsPerSlice + 1] = r1; acc[kDotsPerSlice + 2] = r2; }
      }
      const bool cand = want_hist && slice == 0;
      if (cand) {
        reinterpret_cast<float4*>(yc)[i] = make_float4(yv[0], yv[1], yv[2], yv[3]);
        reinterpret_cast<float4*>(sc)[i] = make_float4(sv[0], sv[1], sv[2], sv[3]);
      }
      {
        float r0 = acc[0], r1 = acc[1], r2 = acc[2], r3 = acc[3];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          r0 += yv[e] * sv[e]; r1 += yv[e] * yv[e];
          r2 += sv[e] * gv[e]; r3 += yv[e] * gv[e];
        }
        if (cand) { acc[0] = r0; acc[1] = r1; acc[2] = r2; acc[3] = r3; }
      }
#pragma unroll
      for (int j = 0; j < kPairsPerSlice; ++j) {
        // predicated loads rather than a branch per pair, so the compiler may issue them ahead of the FFMAs
        const float4 A = (j < nval) ? __ldg(S4 + (int64_t)q[j] * n4 + i) : z4;
        const float4 B = (j < nval) ? __ldg(Y4 + (int64_t)q[j] * n4 + i) : z4;
        const float av[4] = {A.x, A.y, A.z, A.w};
        const float bv[4] = {B.x, B.y, B.z, B.w};
        float r0 = acc[4 + 5 * j], r1 = acc[4 + 5 * j + 1], r2 = acc[4 + 5 * j + 2], r3 = acc[4 + 5 * j + 3],
              r4 = acc[4 + 5 * j + 4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          r0 += av[e] * yv[e];
          r1 += bv[e] * yv[e];
          r2 += sv[e] * bv[e];
          r3 += av[e] * gv[e];
          r4 += bv[e] * gv[e];
        }
        if (j < nval) {  // a pair beyond nval is not added (adding a zero product can turn -0 into +0)
          acc[4 + 5 * j] = r0; acc[4 + 5 * j + 1] = r1; acc[4 + 5 * j + 2] = r2; acc[4 + 5 * j + 3] = r3;
          acc[4 + 5 * j + 4] = r4;
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
  if (last_block_done(&S->ticket)) step_head_body(S, part, gridDim.x, tl, raw, t, count, t_entry, progress);
}

// the vector kernel of a step (see above).  `gz` is the buffer the scatter kernel adds into: g itself
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

// (re)arm the solver for iterations up to `limit`, for the mde_solver_run call numbered `seq`
__global__ void resume_kernel(SolverState* __restrict__ S, int limit, int seq, unsigned long long* progress) {
  if (threadIdx.x != 0) return;
  S->iter_limit = limit;
  if (S->paused && S->iter < limit) { S->paused = 0; S->active = 1; }
  else if (S->active && S->iter >= limit) { S->active = 0; S->paused = 1; }
  set_phase(S, S->phase);
  S->run_seq = seq; S->run_steps = 0;
  publish_progress(progress, S);
}

__global__ void init_state_kernel(SolverState* S, double eps, int memory, int max_stats, int world,
                                  double* avg, double* resid, double* pct, double* steplen) {
  if (threadIdx.x != 0) return;
  S->active = 1; S->converged = 0; S->iter = 0; S->error = 0; S->need_fresh = 1; S->ls_active = 0;
  S->stop_after = 0; S->pad0 = 0; S->eps = eps; S->loss = 0.0; S->gg = 0.0; S->g1 = 0.0;
  S->dd = 0.0; S->xx = 0.0; S->t_last = 0.0; S->t_eval = 0.0; S->func_evals = 0;
  S->max_stats = max_stats; S->world = world;
  S->paused = 0; S->iter_limit = max_stats; S->pend = 0;
  S->run_seq = 0; S->run_steps = 0;
  S->t_cur = 0.0;
  for (int c = 0; c < 4; ++c) { S->cs_g[c] = 0.0; S->cs_d[c] = 0.0; S->mu_x[c] = 0.0f; S->mu_d[c] = 0.0f; }
  for (int q = 0; q < kSlots; ++q) for (int c = 0; c < 4; ++c) { S->cs_S[q][c] = 0.0; S->cs_Y[q][c] = 0.0; }
  set_phase(S, PH_FRESH);  // (sets need_fresh = 1 as well)
  S->ticket = 0u;
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
  unsigned long long* progress = nullptr;      // pinned and mapped: the progress word (host view)
  unsigned long long* progress_dev = nullptr;  //   ... and its device address
  int run_seq = 0;                   // sequence number of the last mde_solver_run call, modulo kProgSeqMask + 1
  long long run_launched = 0;        // steps that call enqueued
  float *X = nullptr, *xinit = nullptr, *d = nullptr, *g = nullptr, *gprev = nullptr, *Sb = nullptr, *Yb = nullptr;
  float* gpart = nullptr;            // multi-GPU: this rank's partial [gradient | loss] before the all-reduce
  double *dpart = nullptr;           // partial rows of the head kernel
  double *vpart = nullptr;           // (g.d, d.d, X.X, max|d|) partials of the vec kernel
  double *stats = nullptr;           // 4 * max_iter doubles
  void* projws = nullptr;
  ProjWs pw{};
  int center_m = 0;                  // {1,2,4}: Centered projection fused into the vec kernel
  int nl = 0;                        // loss-partial blocks of the distortion launch
  int nvb = 0;                       // vector-pass blocks
  int host_active = 0;
  mde_allreduce_fn allreduce = nullptr;
  void* allreduce_user = nullptr;
  // peer-memory all-reduce (world_size > 1): one cudaMalloc region [partial buffer | flags | epoch | ticket],
  // exported with cudaIpc, the peers' regions mapped by mde_solver_comm_connect
  void* comm_region = nullptr;
  int64_t comm_bytes = 0, comm_flags_off = 0, comm_g_off = 0, comm_recv_off = 0, comm_tails_off = 0, comm_slot_floats = 0;
  Comm comm{};
  Comm* comm_dev = nullptr;
  int comm_connected = 0;
  void* peer_base[kMaxWorld] = {nullptr};
  int64_t* anchors = nullptr;
  float* anchor_values = nullptr;
  mde_external_t ext{};              // callable distortion function (ext.d != nullptr), see mde_solver_create_external
  float* gcoef = nullptr;            // (p,) caller-ordered coefficients of the scatter
  int64_t p = 0;
  mde_constraint_part_t cpart{};     // MDE_CONSTRAINT_CUSTOM: the caller's projections, see mde_solver_create_custom
  // stream-launched steps (a caller's part is a hook): the caller's parts that are graphs, instantiated
  // (0 distortion function, 1 retraction, 2 tangent projection)
  cudaGraphExec_t part_exec[3] = {nullptr, nullptr, nullptr};
  // flat step graphs (one step / kStepsPerGraph steps), no conditional nodes
  cudaGraph_t step_graph = nullptr, steps_graph = nullptr;
  cudaGraphExec_t step_exec = nullptr, steps_exec = nullptr;
  int step_kernels = 0;              // kernel nodes per step
  int host_iter = 0;                 // iterations completed (last status read)
  int cur_max_iter = 0;              // iteration cap of the current solve (<= opts.max_iter)
  cudaStream_t cap_stream = nullptr;
};

namespace {

int read_status(mde_solver* s, cudaStream_t st) {
  MDE_CUDA_TRY(cudaMemcpyAsync(s->status_host, s->S, kStatusInts * sizeof(int), cudaMemcpyDeviceToHost, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

// Steps to enqueue now (kStepsPerGraph, 1 or 0), with `in_flight` steps enqueued whose head kernel has not run and
// `left` iterations before the pause, as of one snapshot of the progress word.  An iteration ends in a head kernel and
// takes at least one step, so the next `left` steps all run: an eight-step graph goes in while in_flight + 8 <= left
// (about two of them queued), closer to the pause a one-step graph while in_flight < left (and < 8).  With nothing in
// flight and the solve not stopped, the next step runs too.  So no step is enqueued after the pause.  Near it the queue is one step deep when
// an iteration takes more steps than it has left: the head kernel's result reaches the host while that step's vector
// and distortion kernels run.  (Convergence or an error cannot be foreseen: up to 2 kStepsPerGraph steps are queued
// when one stops the solve, and they exit at their gates.)
int feed_policy(long long in_flight, long long left) {
  if (in_flight <= kStepsPerGraph && in_flight + kStepsPerGraph <= left) return kStepsPerGraph;
  return ((in_flight < left && in_flight < kStepsPerGraph) || in_flight == 0) ? 1 : 0;
}

// Enqueue step graphs as the progress word reports the device's steps, until it reports a stop; *stop = that word.
// Returns with *stop.stopped false when the word has not changed for a second (a step that long, or a stream still
// busy with earlier work): the caller then synchronises and reads the status.  `launched` counts the steps of this run.
int feed_steps(mde_solver* s, int target, int seq, long long* launched, Progress* stop, cudaStream_t st) {
  using clock = std::chrono::steady_clock;
  unsigned long long last = ~0ull;
  clock::time_point since = clock::now();
  *stop = Progress{};
  for (;;) {
    const unsigned long long w = *static_cast<volatile unsigned long long*>(s->progress);
    const Progress pg = decode_progress(w);
    long long done = 0;
    int iter = s->host_iter;
    if (pg.seq == seq) {  // (else resume_kernel of this run has not run yet)
      if (pg.stopped) { *stop = pg; return 0; }
      done = pg.steps;
      iter = pg.iter;
    }
    const int k = feed_policy((*launched - done) & kProgStepsMask, (long long)target - iter);
    if (k) {
      MDE_CUDA_TRY(cudaGraphLaunch(k == 1 ? s->step_exec : s->steps_exec, st));
      *launched += k;
      g_launch_count += (unsigned long long)k * s->step_kernels;
    } else if (w != last) {
      last = w;
      since = clock::now();
    } else if (clock::now() - since > std::chrono::seconds(1)) {
      return 0;
    }
  }
}

// callable distortion function: distances -> the caller's torch code -> coefficients -> scatter.  The caller's part is
// either a CUDA graph, added as a child node of the step graph being captured on `st` (it is not gated: in the surplus
// steps after the device paused it recomputes fpp and loss from a stale d, and nothing reads them), or a host hook
// that enqueues the torch ops on `st` (stream-launched steps).
// the caller's graph inside a step: a child node of the step graph being captured on `st`, after everything captured
// so far; in stream-launched steps (another caller's part is a hook) a launch of its instantiation `exec`
int add_child_graph(cudaGraph_t child, cudaGraphExec_t exec, cudaStream_t st) {
  size_t nodes = 0;
  MDE_CUDA_TRY(cudaGraphGetNodes(child, nullptr, &nodes));
  if (nodes == 0) return 0;  // nothing to do (a tangent projection that returns Z as it is)
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaGraph_t g = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t nd = 0;
  MDE_CUDA_TRY(cudaStreamGetCaptureInfo(st, &cs, nullptr, &g, &deps, &nd));
  if (cs != cudaStreamCaptureStatusActive) {
    if (!exec) return MDE_E_INVALID;
    MDE_CUDA_TRY(cudaGraphLaunch(exec, st));
    return 0;
  }
  cudaGraphNode_t node = nullptr;
  MDE_CUDA_TRY(cudaGraphAddChildGraphNode(&node, g, deps, nd, child));
  MDE_CUDA_TRY(cudaStreamUpdateCaptureDependencies(st, &node, 1, cudaStreamSetCaptureDependencies));
  return 0;
}

int enqueue_external(mde_solver* s, const int* flag, cudaStream_t st) {
  const mde_external_t& x = s->ext;
  int rc = edge_outputs(s->edges, s->X, s->m, x.d, nullptr, flag, st);
  if (rc) return rc;
  if (x.graph) {
    if ((rc = add_child_graph((cudaGraph_t)x.graph, s->part_exec[0], st))) return rc;
  } else {
    if ((rc = x.fn(x.user, x.d, x.fpp, x.loss, (void*)st))) return rc;
  }
  int nb = (int)((s->p + 255) / 256);
  if (nb > kVecBlocks) nb = kVecBlocks;
  ext_coeff_kernel<<<nb, 256, 0, st>>>(flag, x.fpp, x.d, x.loss, s->gcoef, s->edges->loss_partials, s->p);
  MDE_LAUNCH_CHECK();
  return evaluate(2, s->edges, s->X, s->m, s->g, s->gcoef, nullptr, flag, st);
}

// caller-defined constraint: which = 0 retraction [X -> u] -> caller -> [u -> X], which = 1 tangent projection
// [X -> xt, g -> gt] -> caller -> [gt -> g].  The copies are gated on `flag`, the caller's part is not: it only ever
// works on its staging buffers, so in the surplus steps after the device paused it changes nothing the solver (or the
// resumption of a paused solve) reads.
int enqueue_constraint_part(mde_solver* s, int which, const int* flag, cudaStream_t st) {
  const mde_constraint_part_t& c = s->cpart;
  const int64_t n4 = s->npad >> 2;
  const int nb = vec_blocks(n4);
  float* out = which == 0 ? c.u : c.gt;
  gated_copy_kernel<<<nb, kVecThreads, 0, st>>>(flag, s->X, which == 0 ? c.u : c.xt, n4);
  MDE_LAUNCH_CHECK();
  if (which == 1) {
    gated_copy_kernel<<<nb, kVecThreads, 0, st>>>(flag, s->g, c.gt, n4);
    MDE_LAUNCH_CHECK();
  }
  int rc = 0;
  if (c.fn) rc = c.fn(c.user, which, (void*)st);
  else rc = add_child_graph((cudaGraph_t)(which == 0 ? c.retract_graph : c.tangent_graph), s->part_exec[1 + which], st);
  if (rc) return rc;
  gated_copy_kernel<<<nb, kVecThreads, 0, st>>>(flag, out, which == 0 ? s->X : s->g, n4);
  MDE_LAUNCH_CHECK();
  return 0;
}

// closure: value_and_grad at s->X (optim.py:100-105) into the gradient buffer the vec kernel zeroed; `flag` gates
// the kernels.  (g.d, g.g, |g|_1) and the loss are reduced by the next step's head kernel.
int enqueue_eval(mde_solver* s, const int* flag, cudaStream_t st) {
  // several GPUs: scatter into this rank's partial buffer (peer-visible), then all-reduce into g
  const bool multi = s->opts.world_size > 1;
  float* target = multi ? s->gpart : s->g;
  int rc = s->ext.d ? enqueue_external(s, flag, st)
                     : evaluate(0, s->edges, s->X, s->m, target, nullptr, &s->nl, flag, st);
  if (rc) return rc;
  if (multi) {
    pack_loss_kernel<<<1, 256, 0, st>>>(flag, s->edges->loss_partials, s->nl, target + s->npad);
    MDE_LAUNCH_CHECK();
    if (s->comm_connected) {
      const int64_t n4 = s->npad >> 2;
      int nb = (int)((n4 + kCommThreads - 1) / kCommThreads);
      if (nb > kNumSMs) nb = kNumSMs;  // one resident 512-thread block per SM (84-100 registers): a single wave
      if (nb < 1) nb = 1;
      if ((s->npad + 4) * (int64_t)sizeof(float) <= kOneShotBytes) {
        allreduce_kernel<<<nb, kCommThreads, 0, st>>>(flag, s->comm, s->g, s->npad, &s->S->error);
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
      const int64_t n4 = (s->npad + 4) >> 2;
      gated_copy_kernel<<<vec_blocks(n4), kVecThreads, 0, st>>>(flag, s->gpart, s->g, n4);
      MDE_LAUNCH_CHECK();
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
  } else if (s->opts.constraint == MDE_CONSTRAINT_CUSTOM) {
    return enqueue_constraint_part(s, 1, act, st);
  }
  return 0;
}

// one step (see the phase machine above).  Every kernel is gated on the device; the chain has no host decision.
int enqueue_step(mde_solver* s, cudaStream_t st) {
  SolverState* S = s->S;
  int rc = 0;
  const int slices = (s->opts.memory_size + kPairsPerSlice - 1) / kPairsPerSlice;
  Tail tl;
  tl.lpart = s->edges->loss_partials; tl.nl = s->nl; tl.tail = s->g + s->npad;
  tl.p_total = (double)s->edges->p_total; tl.inv_n = 1.0 / (double)s->n;
  step_head_kernel<<<dim3(s->nvb, slices), kVecThreads, 0, st>>>(S, s->g, s->gprev, s->d, s->X, s->Sb, s->Yb, s->npad,
                                                                 s->center_m, s->dpart, s->vpart, tl,
                                                                 s->progress_dev);
  MDE_LAUNCH_CHECK();
  step_vec_kernel<<<s->nvb, kVecThreads, 0, st>>>(S, s->g, s->gprev, s->d, s->X, s->xinit, s->Sb, s->Yb, s->npad,
                                                  s->N, s->center_m, s->opts.world_size > 1 ? s->gpart : s->g,
                                                  s->comm_connected ? s->comm_dev : nullptr, s->vpart);
  MDE_LAUNCH_CHECK();
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
    case MDE_CONSTRAINT_CUSTOM:
      if ((rc = enqueue_constraint_part(s, 0, &S->g_proj, st))) return rc;
      break;
    default: return MDE_E_INVALID;
  }
  return enqueue_eval(s, &S->g_eval, st);
}

int build_step_graph(mde_solver* s, int steps, cudaGraph_t* graph_out, cudaGraphExec_t* exec_out) {
#define GTRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return (int)_e; } while (0)
  if (!s->cap_stream) GTRY(cudaStreamCreateWithFlags(&s->cap_stream, cudaStreamNonBlocking));
  const unsigned long long l0 = g_launch_count;
  if (s->nl == 0) {
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

void destroy_step_graphs(mde_solver* s) {
  if (s->step_exec) cudaGraphExecDestroy(s->step_exec);
  if (s->step_graph) cudaGraphDestroy(s->step_graph);
  if (s->steps_exec) cudaGraphExecDestroy(s->steps_exec);
  if (s->steps_graph) cudaGraphDestroy(s->steps_graph);
  s->step_exec = s->steps_exec = nullptr;
  s->step_graph = s->steps_graph = nullptr;
  for (cudaGraphExec_t& x : s->part_exec) {
    if (x) cudaGraphExecDestroy(x);
    x = nullptr;
  }
}

// the one-step and the kStepsPerGraph-step graphs (one GPU, or several once connected)
int build_step_graphs(mde_solver* s) {
  int rc = build_step_graph(s, 1, &s->step_graph, &s->step_exec);
  if (rc) return rc;
  return build_step_graph(s, kStepsPerGraph, &s->steps_graph, &s->steps_exec);
}

// a graph the solver can embed as a child node: kernel, memset and memcpy nodes only (no memory-allocation nodes);
// an empty one only where `allow_empty`
int check_graph(cudaGraph_t g, bool allow_empty) {
  size_t n = 0;
  MDE_CUDA_TRY(cudaGraphGetNodes(g, nullptr, &n));
  if (n == 0) return allow_empty ? 0 : MDE_E_INVALID;
  cudaGraphNode_t* nodes = new (std::nothrow) cudaGraphNode_t[n];
  if (!nodes) return MDE_E_ALLOC;
  int rc = 0;
  cudaError_t e = cudaGraphGetNodes(g, nodes, &n);
  for (size_t i = 0; e == cudaSuccess && i < n && !rc; ++i) {
    cudaGraphNodeType t;
    e = cudaGraphNodeGetType(nodes[i], &t);
    if (e == cudaSuccess && t != cudaGraphNodeTypeKernel && t != cudaGraphNodeTypeMemset && t != cudaGraphNodeTypeMemcpy)
      rc = MDE_E_UNSUPPORTED;
  }
  delete[] nodes;
  return e != cudaSuccess ? (int)e : rc;
}

int check_external(const mde_external_t* x) {
  if (!x->d || !x->fpp || !x->loss || (!x->graph) == (!x->fn)) return MDE_E_INVALID;
  return x->graph ? check_graph((cudaGraph_t)x->graph, false) : 0;
}

int check_constraint_part(const mde_constraint_part_t* c) {
  const auto misaligned = [](const float* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15u) != 0; };
  if (misaligned(c->u) || misaligned(c->xt) || misaligned(c->gt)) return MDE_E_INVALID;
  if ((!c->retract_graph) != (!c->tangent_graph)) return MDE_E_INVALID;  // both graphs, or none
  if ((!c->retract_graph) == (!c->fn)) return MDE_E_INVALID;             // graphs or a hook
  if (c->fn) return 0;
  const int rc = check_graph((cudaGraph_t)c->retract_graph, true);
  return rc ? rc : check_graph((cudaGraph_t)c->tangent_graph, true);
}

// (re)build the step graphs around the caller's parts: when every part is a graph the steps are captured with those
// graphs inside; when any part is a hook the steps are stream-launched, there are no step graphs, and the parts that
// are graphs are instantiated to be launched inside those steps
int rebuild_step_graphs(mde_solver* s) {
  destroy_step_graphs(s);
  const bool hook = (s->ext.d && !s->ext.graph) || s->cpart.fn;
  if (!hook) return build_step_graphs(s);
  const void* parts[3] = {s->ext.graph, s->cpart.retract_graph, s->cpart.tangent_graph};
  for (int k = 0; k < 3; ++k) {
    size_t nodes = 0;
    if (parts[k]) MDE_CUDA_TRY(cudaGraphGetNodes((cudaGraph_t)parts[k], nullptr, &nodes));
    if (nodes) MDE_CUDA_TRY(cudaGraphInstantiate(&s->part_exec[k], (cudaGraph_t)parts[k], 0));
  }
  return 0;
}

int attach_external(mde_solver* s, const mde_external_t* x) {
  s->ext = *x;
  s->nl = 1;  // the loss arrives as one partial (ext_coeff_kernel)
  return rebuild_step_graphs(s);
}

int solver_create(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m, const mde_solver_opts_t* opts,
                  const mde_external_t* ext, const mde_constraint_part_t* cpart, void* stream) {
  if (!out || !e || !opts || n < 1 || m < 1) return MDE_E_INVALID;
  if (opts->memory_size < 1 || opts->memory_size > kMaxMemory) return MDE_E_UNSUPPORTED;
  if (opts->constraint < 0 || opts->constraint > MDE_CONSTRAINT_CUSTOM) return MDE_E_INVALID;
  if ((opts->constraint == MDE_CONSTRAINT_CUSTOM) != (cpart != nullptr)) return MDE_E_INVALID;
  if (opts->max_iter < 1) return MDE_E_INVALID;
  if (opts->mode == 0 || opts->mode == 1) return MDE_E_UNSUPPORTED;  // retired drivers (host-stepped, conditional graph)
  if (opts->mode != 2) return MDE_E_INVALID;
  if (n != e->n) return MDE_E_INVALID;
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
  TRY(cudaHostAlloc(&s->progress, sizeof(unsigned long long), cudaHostAllocMapped));
  *s->progress = 0ull;
  TRY(cudaHostGetDevicePointer(&s->progress_dev, s->progress, 0));
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
  if (cpart) s->cpart = *cpart;  // (before the first capture, like the external descriptor)
  if (ext) {  // the descriptor is in place before the first capture
    s->p = e->p;
    TRY(cudaMalloc(&s->gcoef, sizeof(float) * s->p));
    TRY(cudaStreamSynchronize(st));
    if ((rc = attach_external(s, ext))) goto fail;
  } else if (cpart) {
    s->nl = 0;
    TRY(cudaStreamSynchronize(st));
    if ((rc = rebuild_step_graphs(s))) goto fail;
  } else if (opts->world_size == 1) {  // several GPUs: graphs are built by mde_solver_comm_connect
    s->nl = 0;
    TRY(cudaStreamSynchronize(st));
    if ((rc = build_step_graphs(s))) goto fail;
  }
  *out = s;
  return 0;
fail:
  mde_solver_destroy(s);
  return rc;
#undef TRY
}

}  // namespace

extern "C" {

int mde_solver_create(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m, const mde_solver_opts_t* opts,
                      void* stream) {
  return solver_create(out, e, n, m, opts, nullptr, nullptr, stream);
}

int mde_solver_create_external(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m,
                               const mde_solver_opts_t* opts, const mde_external_t* ext, void* stream) {
  if (!ext || !opts || opts->world_size != 1) return MDE_E_INVALID;
  const int rc = check_external(ext);
  if (rc) return rc;
  return solver_create(out, e, n, m, opts, ext, nullptr, stream);
}

int mde_solver_create_custom(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m,
                             const mde_solver_opts_t* opts, const mde_external_t* ext,
                             const mde_constraint_part_t* part, void* stream) {
  if (!out || !e || !part || !opts || opts->world_size != 1 || opts->constraint != MDE_CONSTRAINT_CUSTOM)
    return MDE_E_INVALID;
  int rc = check_constraint_part(part);
  if (rc) return rc;
  if (ext && (rc = check_external(ext))) return rc;
  return solver_create(out, e, n, m, opts, ext, part, stream);
}

int mde_solver_set_constraint_part(mde_solver_t* s, const mde_constraint_part_t* part, void* stream) {
  if (!s || !part || s->opts.constraint != MDE_CONSTRAINT_CUSTOM) return MDE_E_INVALID;
  int rc = check_constraint_part(part);
  if (rc) return rc;
  MDE_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));  // no step that embeds the old part is in flight
  s->cpart = *part;
  return rebuild_step_graphs(s);
}

int mde_solver_set_external(mde_solver_t* s, const mde_external_t* ext, void* stream) {
  if (!s || !ext || !s->ext.d) return MDE_E_INVALID;
  int rc = check_external(ext);
  if (rc) return rc;
  MDE_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));  // no step that embeds the old part is in flight
  return attach_external(s, ext);
}

int mde_solver_destroy(mde_solver_t* s) {
  if (!s) return 0;
  cudaFree(s->S); cudaFreeHost(s->status_host); cudaFreeHost(s->progress);
  cudaFree(s->X); cudaFree(s->xinit); cudaFree(s->d); cudaFree(s->gprev);
  if (!s->comm_region) cudaFree(s->g);  // (several GPUs: g lives inside the peer-visible region)
  for (int q = 0; q < kMaxWorld; ++q) if (s->peer_base[q]) cudaIpcCloseMemHandle(s->peer_base[q]);
  cudaFree(s->comm_region); cudaFree(s->comm_dev);
  cudaFree(s->Sb); cudaFree(s->Yb); cudaFree(s->dpart); cudaFree(s->vpart); cudaFree(s->stats); cudaFree(s->projws);
  cudaFree(s->anchors); cudaFree(s->anchor_values); cudaFree(s->gcoef);
  destroy_step_graphs(s);
  if (s->cap_stream) cudaStreamDestroy(s->cap_stream);
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
  // the sharded solve runs the same flat step graphs as one GPU
  s->nl = 0;
  return build_step_graphs(s);
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
  s->host_active = 1;
  s->host_iter = 0;
  return 0;
}

// globaltimer stamps (ns) of the last head kernel that started an iteration: [0] last block's entry,
// [1] epilogue entry, [2] state staged, [3] partials reduced, [4] previous step finished, [5] direction done,
// [6] before write-back, [7] the vec kernel's first block.  Diagnostics only (tools/solver_times.py).
int mde_solver_debug_times(mde_solver_t* s, unsigned long long* out8, void* stream) {
  if (!s || !out8) return MDE_E_INVALID;
  MDE_CUDA_TRY(cudaMemcpyAsync(out8, s->S->dbg, sizeof(unsigned long long) * 8, cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  MDE_CUDA_TRY(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

// L-BFGS state of a paused solve, copied as it is (no kernel, no device write): the gradient buffer, g_prev and d of
// the last completed iteration, the stored pairs in logical order (slot order[j], first n*m floats), H_diag, n_iter.
// Diagnostics only (tests/test_gpu_lbfgs_replay.py replays the solve from these in fp64).
int mde_solver_debug_lbfgs(mde_solver_t* s, float* g, float* g_prev, float* d, float* S_out, float* Y_out, int* count,
                           double* h_diag, int* n_iter, void* stream) {
  if (!s || !g || !g_prev || !d || !S_out || !Y_out || !count || !h_diag || !n_iter) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = read_status(s, st);
  if (rc) return rc;
  if (!s->host_active || !s->status_host[8]) return MDE_E_INVALID;  // only between two runs of a paused solve
  LbfgsState* lb = new (std::nothrow) LbfgsState();
  if (!lb) return MDE_E_ALLOC;
  const size_t vb = sizeof(float) * (size_t)s->N;
  cudaError_t e = cudaMemcpyAsync(lb, (const char*)s->S + offsetof(SolverState, lb), sizeof(LbfgsState),
                                  cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(g, s->g, vb, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(g_prev, s->gprev, vb, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d, s->d, vb, cudaMemcpyDeviceToHost, st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  for (int j = 0; e == cudaSuccess && j < lb->count; ++j) {
    const int64_t q = lb->order[j];
    e = cudaMemcpyAsync(S_out + (int64_t)j * s->N, s->Sb + q * s->npad, vb, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(Y_out + (int64_t)j * s->N, s->Yb + q * s->npad, vb, cudaMemcpyDeviceToHost, st);
  }
  if (e == cudaSuccess) e = cudaStreamSynchronize(st);
  *count = lb->count; *h_diag = lb->H_diag; *n_iter = lb->n_iter;
  delete lb;
  return e == cudaSuccess ? 0 : (int)e;
}

int mde_solver_run(mde_solver_t* s, int iters, int* iters_done, int* converged, void* stream) {
  if (!s) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = 0;
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
  const int seq = s->run_seq = (s->run_seq + 1) & kProgSeqMask;
  resume_kernel<<<1, 32, 0, st>>>(s->S, target, seq, s->progress_dev);
  MDE_LAUNCH_CHECK();
  // One GPU with step graphs: the host keeps the queue fed from the progress word and takes the result of a clean stop
  // (pause, convergence, iteration cap) from it, without synchronising: what is still queued then is the rest of the
  // stopping step and the steps after a convergence, all gated off, and they complete in stream order.  After an
  // error or a stall it reads the status.  Stream-launched steps and sharded solves read the status after every
  // batch (every rank must enqueue the same steps, decided from the same status).
  const bool fed = s->steps_exec && s->opts.world_size == 1;
  long long launched = 0;
  for (int round = 0;; ++round) {
    if (round > (1 << 18)) return MDE_E_INVALID;
    int remaining = target - s->host_iter;
    if (remaining < 1) remaining = 1;
    long long steps = 0;
    if (fed) {
      Progress stop;
      rc = feed_steps(s, target, seq, &launched, &stop, st);
      s->run_launched = launched;
      if (rc) return rc;
      if (stop.stopped && !stop.failed) {
        s->host_iter = stop.iter;
        s->host_active = stop.paused;  // only a pause can be resumed
        if (iters_done) *iters_done = stop.iter;
        if (converged) *converged = stop.converged;
        return 0;
      }
    } else if (!s->steps_exec) {
      // host hook (all-reduce, or a callable distortion function in hook mode): stream-launched steps; every rank
      // enqueues the same number of steps (same `remaining`: the replicated state machines agree)
      int n_steps = remaining + remaining / 8 + (round > 0 ? 1 : 0) + 1;
      if (n_steps > 64) n_steps = 64;
      for (int b = 0; b < n_steps; ++b) { if ((rc = enqueue_step(s, st))) return rc; }
      launched += n_steps;
    } else if (remaining >= kStepsPerGraph) {
      int graphs = (remaining + remaining / 8 + 1) / kStepsPerGraph;
      if (graphs * kStepsPerGraph > 96) graphs = 96 / kStepsPerGraph;  // <= ~96 steps in flight per status read
      for (int b = 0; b < graphs; ++b) MDE_CUDA_TRY(cudaGraphLaunch(s->steps_exec, st));
      steps = (long long)graphs * kStepsPerGraph;
    } else {
      const int singles = remaining + remaining / 4 + (round > 0 ? 1 : 0) + 1;
      for (int b = 0; b < singles; ++b) MDE_CUDA_TRY(cudaGraphLaunch(s->step_exec, st));
      steps = singles;
    }
    g_launch_count += (unsigned long long)steps * s->step_kernels;  // (stream-launched steps count themselves)
    launched += steps;
    s->run_launched = launched;
    if ((rc = read_status(s, st))) return rc;
    s->host_iter = s->status_host[2];
    if (s->status_host[3]) { s->host_active = 0; if (iters_done) *iters_done = s->status_host[2]; return s->status_host[3]; }
    if (!s->status_host[0]) {              // paused at the target, converged, or out of iterations
      s->host_active = s->status_host[8];  // only a pause can be resumed
      break;
    }
    // still active after a stall: every step enqueued has run, and each one published the word
    const Progress pg = decode_progress(*static_cast<volatile unsigned long long*>(s->progress));
    if (fed && (pg.seq != seq || pg.steps != (launched & kProgStepsMask))) return MDE_E_INVALID;
  }
  if (iters_done) *iters_done = s->status_host[2];
  if (converged) *converged = s->status_host[1];
  return 0;
}

int mde_solver_debug_run_steps(mde_solver_t* s, int64_t* launched, int64_t* ran) {
  if (!s || !launched || !ran) return MDE_E_INVALID;
  const Progress pg = decode_progress(*static_cast<volatile unsigned long long*>(s->progress));
  *launched = s->run_launched;
  *ran = pg.seq == s->run_seq ? pg.steps : 0;
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
int mde_dbg_feed_policy(int64_t in_flight, int64_t left) { return feed_policy(in_flight, left); }
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
