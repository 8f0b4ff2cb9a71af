// mde_edges.cu -- edge layout + the fused average-distortion kernel (forward + backward), the evaluation entries that
// pick the kernels of every layout kind, and the launch helpers the tile, pull and ELL layouts share (mde_edges.cuh).
//
// Replaces pymde/average_distortion.py:36-80 (gather X[lhs], X[rhs]; row norms; per-edge
// penalty; mean; scatter-add of +-g*diff) and pymde/problem.py:246-307 (per-edge outputs).
//
// Data layout in HBM (one shard):
//   src[p], dst[p]  int32   canonical (src < dst) endpoints, sorted by (class, src, dst)
//                           class 0 = attractive/ordinary, 1 = repulsive (PushAndPull w < 0)
//   par0[p]         fp32    weight | deviation, permuted alongside
//   par1[p]         fp32    optional second array (WeightedQuadratic weights)
//   perm[p]         int32   original position of sorted edge k (per-edge outputs only)
// Algorithmic bytes per fused evaluation: p*(8+4k) + 2*n*m*4 + 8  (SURVEY section 8d).
//
// Kernel shapes
//   m <= 4, default (fused value + gradient and external coefficients): distortion_owner_kernel walks the directed
//            entries `ent` grouped by owner node, 8 lanes per node, sum in registers, one write per row, no atomics.
//   m <= 4, value only / MDE_B200_DETERMINISTIC / other m: one thread per edge (quad or strided kernel); the lhs
//            contributions (sorted => runs of equal src) are summed with a warp segmented
//            reduction and issued as ONE vector red per run; rhs contributions go out as
//            vector reds (REDG.E.ADD.F32x2/x4).
//   m >= 5 : a group of G lanes (8/16/32) walks a contiguous slice of edges; the lhs row and
//            its gradient accumulator stay in registers across a run.
//   5 <= m <= 512, MDE_B200_DETERMINISTIC (fused and external coefficients): distortion_wide_owner_kernel, one group
//            of G lanes per owner over its directed entries `ent`, one write per row, no atomics.
#include <cub/cub.cuh>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <new>
#include <utility>

#include "mde_edges.cuh"

namespace mde {
unsigned long long g_launch_count = 0;
}

using namespace mde;

static constexpr int kSmallThreads = 256;
static constexpr int kRounds = 4;  // 32-edge rounds per warp iteration

// ------------------------------------------------------------------------------------------
// layout build
// ------------------------------------------------------------------------------------------
__global__ void make_keys_kernel(const int64_t* __restrict__ edges, const float* __restrict__ par0,
                                 int push_pull, int64_t p, uint64_t* __restrict__ keys,
                                 int32_t* __restrict__ vals) {
  int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p) return;
  int64_t i = edges[2 * k], j = edges[2 * k + 1];
  uint64_t lo = (uint64_t)(i < j ? i : j), hi = (uint64_t)(i < j ? j : i);
  uint64_t cls = (push_pull && !(par0[k] >= 0.0f)) ? 1ull : 0ull;
  keys[k] = (cls << 63) | (lo << 32) | hi;  // n < 2^31
  vals[k] = (int32_t)k;
}

__global__ void unpack_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals,
                              const float* __restrict__ par0, const float* __restrict__ par1, int64_t p,
                              int32_t* __restrict__ src, int32_t* __restrict__ dst,
                              float* __restrict__ p0, float* __restrict__ p1, int32_t* __restrict__ perm) {
  int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t p4 = (p + 3) & ~(int64_t)3;  // arrays are padded to a multiple of 4 edges
  if (k >= p4) return;
  const int64_t kk = k < p ? k : p - 1;     // pad entries repeat the last edge (masked in the kernels)
  uint64_t key = keys[kk];
  src[k] = (int32_t)((key >> 32) & 0x7fffffffu);
  dst[k] = (int32_t)(key & 0xffffffffu);
  int32_t o = vals[kk];
  p0[k] = par0[o];
  if (par1) p1[k] = par1[o];
  perm[k] = o;  // padded like the other arrays: the quad kernel loads it as int4 (MODE 2)
}

// ------------------------------------------------------------------------------------------
// m <= 4: thread-per-edge kernel
// ------------------------------------------------------------------------------------------
// Deterministic mode: contributions are accumulated as 64-bit fixed point (scale 2^40, resolution 9e-13, range
// +-8.4e6 -- the entries are f'/p-sized).  Integer addition is associative, so the sums do not depend on the order in
// which the reds land (the float reds of the default mode, like the reference's scatter_add_, do:
// pymde/average_distortion.py:75-76).
constexpr float kFxScale = 1099511627776.0f;  // 2^40
template <int M>
__device__ __forceinline__ void red_row_fx(long long* __restrict__ F, int r, const float (&v)[M], float sgn) {
#pragma unroll
  for (int c = 0; c < M; ++c) {
    const long long q = __float2ll_rn(sgn * v[c] * kFxScale);
    atomicAdd(reinterpret_cast<unsigned long long*>(F + (int64_t)r * M + c), (unsigned long long)q);
  }
}
// incidence entries of the sorted edges: (node, (k << 1) | endpoint is dst); the per-node counts on the side
__global__ void inc_keys_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst, int64_t p,
                                uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, int* __restrict__ count) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 2 * p) return;
  const int64_t k = j < p ? j : j - p;
  const int node = j < p ? src[k] : dst[k];
  keys[j] = (uint32_t)node;
  vals[j] = ((uint32_t)k << 1) | (j < p ? 0u : 1u);
  atomicAdd(count + node, 1);
}
// directed entries in the order of `inc`: (neighbour row | endpoint is dst << 31, bits of par0[k])
__global__ void ent_fill_kernel(const uint32_t* __restrict__ inc, const int32_t* __restrict__ src,
                                const int32_t* __restrict__ dst, const float* __restrict__ par0, int64_t q,
                                uint2* __restrict__ ent) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= q) return;
  const uint32_t w = inc[j];
  const int64_t k = (int64_t)(w >> 1);
  const uint32_t is_dst = w & 1u;
  const uint32_t nbr = (uint32_t)(is_dst ? src[k] : dst[k]);
  ent[j] = make_uint2(nbr | (is_dst << 31), __float_as_uint(par0[k]));
}
__global__ void fx_zero_kernel(const int* __restrict__ flag, long long* __restrict__ F, int64_t count) {
  if (flag != nullptr && *flag == 0) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride) F[i] = 0ll;
}
__global__ void fx_apply_kernel(const int* __restrict__ flag, const long long* __restrict__ F, float* __restrict__ grad,
                                int64_t count) {
  if (flag != nullptr && *flag == 0) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
    grad[i] += (float)((double)F[i] * (1.0 / 1099511627776.0));
}

// MODE 0: fused value + gradient; 1: value only; 2: external per-edge g (gradient only)
template <int M, int MODE, int FA, int FR>
__global__ void __launch_bounds__(kSmallThreads)
distortion_small_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                        const float* __restrict__ par0, const float* __restrict__ par1,
                        const int32_t* __restrict__ perm, const float* __restrict__ gext,
                        int64_t p, const float* __restrict__ X, float* __restrict__ grad,
                        double* __restrict__ loss_partials, FnDev fn, float inv_p,
                        const int* __restrict__ flag) {
  if (flag != nullptr && *flag == 0) return;
  const int lane = threadIdx.x & 31;
  const int64_t warp0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nwarps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  constexpr int64_t kPerWarp = 32 * kRounds;
  double lsum = 0.0;

  for (int64_t base = warp0 * kPerWarp; base < p; base += nwarps * kPerWarp) {
    int s[kRounds], t[kRounds];
    float a[kRounds], b[kRounds];
    bool ok[kRounds];
    // Out-of-range lanes re-read the last edge (index clamp) instead of selecting zeros: every lane
    // then holds valid row indices and no address is formed from a predicated value.
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
      int64_t k = base + r * 32 + lane;
      ok[r] = k < p;
      const int64_t kk = ok[r] ? k : (p - 1);
      s[r] = __ldg(src + kk);
      t[r] = __ldg(dst + kk);
      if (MODE == 2) a[r] = __ldg(gext + __ldg(perm + kk));
      else a[r] = __ldg(par0 + kk);
      b[r] = (MODE != 2 && par1 != nullptr) ? __ldg(par1 + kk) : 0.0f;
    }
    Row<M> xi[kRounds], xj[kRounds];
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
      xi[r] = ldg_row<M>(X, s[r]);
      xj[r] = ldg_row<M>(X, t[r]);
    }
#pragma unroll
    for (int r = 0; r < kRounds; ++r) {
      float diff[M];
      float d2 = 0.0f;
#pragma unroll
      for (int c = 0; c < M; ++c) { diff[c] = xi[r].v[c] - xj[r].v[c]; d2 += diff[c] * diff[c]; }
      float g;
      if (MODE == 2) {
        g = a[r];
      } else {
        float d = sqrtf(d2), f;
        if (MODE == 0) edge_coeff<FA, FR>(fn, d, a[r], b[r], inv_p, f, g);
        else { edge_value<FA, FR>(fn, d, a[r], b[r], f); g = 0.0f; }
        if (ok[r]) lsum += (double)f;
      }
      if (MODE != 1) {
        float v[M];
#pragma unroll
        for (int c = 0; c < M; ++c) v[c] = ok[r] ? g * diff[c] : 0.0f;
        if (ok[r]) red_row<M>(grad, t[r], v, -1.0f);
        // lhs: sorted => equal keys are adjacent lanes; segmented warp reduction
        int key = ok[r] ? s[r] : (-1 - lane);
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
          int k2 = __shfl_down_sync(kFull, key, off);
          bool take = (lane + off < 32) && (k2 == key);
#pragma unroll
          for (int c = 0; c < M; ++c) {
            float o = __shfl_down_sync(kFull, v[c], off);
            if (take) v[c] += o;
          }
        }
        int kprev = __shfl_up_sync(kFull, key, 1);
        bool head = (lane == 0) || (kprev != key);
        if (head && ok[r]) red_row<M>(grad, s[r], v, 1.0f);
      }
    }
  }
  if (MODE != 2) {
    __shared__ double sm[32];
    double v1[1] = {lsum};
    block_sum<1>(v1, sm);
    if (threadIdx.x == 0) loss_partials[blockIdx.x] = v1[0];
  }
}

// ------------------------------------------------------------------------------------------
// m <= 4, thread-contiguous variant: each thread owns 4 CONSECUTIVE sorted edges (three 16-byte
// loads for src/dst/par0), sums the lhs contributions of equal-src runs in registers and issues one
// red per run; no warp shuffles.  FAST selects the MUFU-based math for PushAndPull(Log1p(1.5), Log(1)).
// ------------------------------------------------------------------------------------------
static constexpr int kQuadThreads = 256;

// One edge's loss term f and gradient contribution v = g (x_src - x_dst) (added at src, subtracted at dst).  The quad
// kernel and the owner kernel both evaluate edges through this function, so they produce the same floats.  MODE 2
// takes g = a; MODE 1 leaves v unset.  d = 0: the reference replaces the non-finite g by 1 and the difference vector
// is 0.  Returns whether v is live (v = 0 otherwise).  `v` must be rounded on its own before it is summed: the owner
// kernel adds it with __fadd_rn, so that no contraction fuses g * diff into the accumulation.
template <int M, int MODE, int FA, int FR, bool FAST>
__device__ __forceinline__ bool edge_contribution(const Row<M>& xs, const Row<M>& xd, float a, float b, const FnDev& fn,
                                                  float inv_p, bool ok, float& f, float (&v)[M]) {
  float diff[M];
  float d2 = 0.0f;
#pragma unroll
  for (int c = 0; c < M; ++c) { diff[c] = xs.v[c] - xd.v[c]; d2 += diff[c] * diff[c]; }
  float g;
  f = 0.0f;
  if (MODE == 2) {
    g = a;
  } else if (FAST) {
    edge_coeff_fast_log1p_log<2>(d2, a, inv_p, f, g);
  } else {
    const float d = sqrtf(d2);
    if (MODE == 0) edge_coeff<FA, FR>(fn, d, a, b, inv_p, f, g);
    else { edge_value<FA, FR>(fn, d, a, b, f); g = 0.0f; }
  }
  const bool live = ok && (FAST ? (d2 > 0.0f) : true);
  if (MODE != 1) {
#pragma unroll
    for (int c = 0; c < M; ++c) v[c] = live ? g * diff[c] : 0.0f;
  }
  return live;
}

template <int M, int MODE, int FA, int FR, bool FAST, int NQ>
__global__ void __launch_bounds__(kQuadThreads)
distortion_quad_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                       const float* __restrict__ par0, const float* __restrict__ par1,
                       const int32_t* __restrict__ perm, const float* __restrict__ gext,
                       int64_t p, const float* __restrict__ X, float* __restrict__ grad,
                       double* __restrict__ loss_partials, FnDev fn, float inv_p,
                       const int* __restrict__ flag, long long* __restrict__ fx) {
  if (flag != nullptr && *flag == 0) return;
  constexpr int E = 4 * NQ;  // consecutive edges owned by a thread per iteration
  const int64_t nquads = (p + 3) >> 2;
  const int64_t nunits = (nquads + NQ - 1) / NQ;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  float lsum_f = 0.0f;
  double lsum = 0.0;
  // software pipeline (NQ == 1): the edge record of the NEXT grid-stride iteration is requested before the
  // vertex rows of the current one are gathered, so its latency overlaps the gathers and the math
  int4 s4n = make_int4(0, 0, 0, 0), t4n = make_int4(0, 0, 0, 0);
  float4 a4n = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool pipe = (NQ == 1 && MODE != 2);
  {
    const int64_t u0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (pipe && u0 < nunits) {
      s4n = __ldg(reinterpret_cast<const int4*>(src) + u0);
      t4n = __ldg(reinterpret_cast<const int4*>(dst) + u0);
      a4n = __ldg(reinterpret_cast<const float4*>(par0) + u0);
    }
  }
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < nunits; u += stride) {
    int s[E], t[E];
    float a[E], b[E];
#pragma unroll
    for (int j = 0; j < NQ; ++j) {
      const int64_t q = u * NQ + j;
      const int64_t qc = q < nquads ? q : nquads - 1;  // clamped: masked below through `ok`
      int4 s4, t4;
      if (pipe) {
        s4 = s4n; t4 = t4n;
        const int64_t un = u + stride;
        if (un < nunits) {
          s4n = __ldg(reinterpret_cast<const int4*>(src) + un);
          t4n = __ldg(reinterpret_cast<const int4*>(dst) + un);
        }
      } else {
        s4 = __ldg(reinterpret_cast<const int4*>(src) + qc);
        t4 = __ldg(reinterpret_cast<const int4*>(dst) + qc);
      }
      s[4 * j] = s4.x; s[4 * j + 1] = s4.y; s[4 * j + 2] = s4.z; s[4 * j + 3] = s4.w;
      t[4 * j] = t4.x; t[4 * j + 1] = t4.y; t[4 * j + 2] = t4.z; t[4 * j + 3] = t4.w;
      if (MODE == 2) {
        const int4 o4 = __ldg(reinterpret_cast<const int4*>(perm) + qc);  // pad entries repeat the last edge
        a[4 * j] = __ldg(gext + o4.x); a[4 * j + 1] = __ldg(gext + o4.y);
        a[4 * j + 2] = __ldg(gext + o4.z); a[4 * j + 3] = __ldg(gext + o4.w);
      } else {
        float4 a4;
        if (pipe) {
          a4 = a4n;
          const int64_t un = u + stride;
          if (un < nunits) a4n = __ldg(reinterpret_cast<const float4*>(par0) + un);
        } else {
          a4 = __ldg(reinterpret_cast<const float4*>(par0) + qc);
        }
        a[4 * j] = a4.x; a[4 * j + 1] = a4.y; a[4 * j + 2] = a4.z; a[4 * j + 3] = a4.w;
      }
      if (MODE != 2 && par1 != nullptr) {
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(par1) + qc);
        b[4 * j] = b4.x; b[4 * j + 1] = b4.y; b[4 * j + 2] = b4.z; b[4 * j + 3] = b4.w;
      } else { b[4 * j] = b[4 * j + 1] = b[4 * j + 2] = b[4 * j + 3] = 0.0f; }
    }
    Row<M> xi[E], xj[E];
#pragma unroll
    for (int e = 0; e < E; ++e) { xi[e] = ldg_row<M>(X, s[e]); xj[e] = ldg_row<M>(X, t[e]); }
    float acc[M];
#pragma unroll
    for (int c = 0; c < M; ++c) acc[c] = 0.0f;
    int cur = s[0];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const bool ok = (4 * (u * NQ) + e) < p;
      float f, v[M];
      const bool live = edge_contribution<M, MODE, FA, FR, FAST>(xi[e], xj[e], a[e], b[e], fn, inv_p, ok, f, v);
      if (MODE != 2 && ok) { if (FAST) lsum_f += f; else lsum += (double)f; }
      if (MODE != 1) {
        if (live) { if (fx) red_row_fx<M>(fx, t[e], v, -1.0f); else red_row<M>(grad, t[e], v, -1.0f); }
        if (s[e] != cur) {  // run of equal src ended: flush its sum
          if (fx) red_row_fx<M>(fx, cur, acc, 1.0f); else red_row<M>(grad, cur, acc, 1.0f);
          cur = s[e];
#pragma unroll
          for (int c = 0; c < M; ++c) acc[c] = 0.0f;
        }
#pragma unroll
        for (int c = 0; c < M; ++c) acc[c] += v[c];
      }
    }
    if (MODE != 1) { if (fx) red_row_fx<M>(fx, cur, acc, 1.0f); else red_row<M>(grad, cur, acc, 1.0f); }
    if (FAST) { lsum += (double)lsum_f; lsum_f = 0.0f; }
  }
  if (MODE != 2) {
    __shared__ double sm[32];
    double v1[1] = {lsum};
    block_sum<1>(v1, sm);
    if (threadIdx.x == 0) loss_partials[blockIdx.x] = v1[0];
  }
}

// ------------------------------------------------------------------------------------------
// m <= 4, owner-complete pass over the directed entries of the sorted-SoA layout (MODE 0 and 2).  kOwnerLanes lanes
// per node: lane l evaluates the entries l, l + 8, ... of the node's list in order and keeps their sum in registers,
// the lanes are combined by a fixed shuffle tree and the row is written once.  Every edge is evaluated at both of its
// ends, with the same operands, so each contribution is the same float at both; no atomics and no second pass, so
// the gradient is the same bits in every run.  The loss counts each edge once, at its src-end entry, in fp64.
// ------------------------------------------------------------------------------------------
static constexpr int kOwnerLanes = 8;
static constexpr int kOwnerThreads = 256;
static constexpr int kOwnerNodes = kOwnerThreads / kOwnerLanes;  // nodes per block and trip
static constexpr int kOwnerBatch = 4;  // entries per lane whose loads are issued before the first of them is added
static constexpr int kOwnerHub = 128;  // longer lists are evaluated by the whole warp (same entries per lane, same order)
// Resident blocks per SM that the register allocation must allow.  The grid is two waves at 8 blocks per SM
// (loss_blocks_owner).  The MUFU kernel at m = 2 fits 6 blocks (40 registers) without spilling, where the compiler's
// own choice of 43 leaves 5; 8 blocks (32 registers) spill and measured slower.  Every other instantiation keeps the
// compiler's allocation.
template <int M, bool FAST>
constexpr int owner_min_blocks() { return (FAST && M == 2) ? 6 : 1; }

template <int M, int MODE, int FA, int FR, bool FAST>
__global__ void __launch_bounds__(kOwnerThreads, owner_min_blocks<M, FAST>())
distortion_owner_kernel(const uint2* __restrict__ ent, const uint32_t* __restrict__ inc,
                        const int64_t* __restrict__ off, const float* __restrict__ par1,
                        const int32_t* __restrict__ perm, const float* __restrict__ gext, int64_t n,
                        const float* __restrict__ X, float* __restrict__ grad, double* __restrict__ loss_partials,
                        FnDev fn, float inv_p, const int* __restrict__ flag) {
  static_assert(MODE == 0 || MODE == 2, "value-only evaluations run on the quad kernel");
  if (flag != nullptr && *flag == 0) return;
  const int lane = threadIdx.x & 31, l = lane % kOwnerLanes;
  // par1[k] and gext[perm[k]] are indexed by the sorted edge.  Of the compile-time functions only WeightedQuadratic
  // reads its second parameter, so every other pair compiles the lookup out.
  constexpr bool kReadsPar1 = FA < 0 || FA == MDE_FN_L_WEIGHTED_QUADRATIC || FR == MDE_FN_L_WEIGHTED_QUADRATIC;
  const bool need_k = MODE == 2 || (kReadsPar1 && par1 != nullptr);
  double lsum = 0.0;
  // one entry: record w (w.y holds the coefficient a, the caller's in MODE 2) and second parameter b.  Past the end
  // of a list nothing is loaded.  The records are read once per evaluation: ldg_stream.  Entry indices fit in int:
  // the layout needs 2 p < 2^31.
  auto fetch = [&](int j, bool in, uint2& w, float& b) {
    w = make_uint2(0u, 0u);
    b = 0.0f;
    if (in) {
      w = ldg_stream(ent + j);
      if (need_k) {
        const uint32_t k = ldg_stream(inc + j) >> 1;
        if (MODE == 2) w.y = __float_as_uint(__ldg(gext + __ldg(perm + k)));
        else b = __ldg(par1 + k);
      }
    }
  };
  // the neighbour's row of a fetched entry; past the end of a list no gather is issued (the value is never used)
  auto gather = [&](uint2 w, bool in, const Row<M>& xo) {
    return in ? ldg_row<M>(X, (int)(w.x & 0x7fffffffu)) : xo;
  };
  // The signed contribution of an entry to the owner's row.  The edge's difference is x_src - x_dst at both ends and
  // the owner adds +v at the src end, -v at the dst end; rounding is symmetric in sign, so that is g (x_owner -
  // x_neighbour) at either end, with the same d2, f and g.  The loss counts the edge at its src end.
  auto contribution = [&](const Row<M>& xo, const Row<M>& xn, uint2 w, float b, bool in, float (&v)[M]) {
    float f;
    edge_contribution<M, MODE, FA, FR, FAST>(xo, xn, __uint_as_float(w.y), b, fn, inv_p, true, f, v);
    if (MODE != 2 && in && (w.x >> 31) == 0) lsum += (double)f;
  };
  // the trip count is uniform across the block: the shuffles and the block sum need every lane
  for (int64_t i0 = (int64_t)blockIdx.x * kOwnerNodes; i0 < n; i0 += (int64_t)gridDim.x * kOwnerNodes) {
    const int64_t il = i0 + threadIdx.x / kOwnerLanes;
    const bool node = il < n;
    const int i = node ? (int)il : 0;
    float acc[M];
#pragma unroll
    for (int c = 0; c < M; ++c) acc[c] = 0.0f;
    const int j0 = node ? (int)ldg_stream(off + i) : 0, cnt = node ? (int)ldg_stream(off + i + 1) - j0 : 0;
    const bool hub = cnt > kOwnerHub;
    if (node && !hub) {
      const Row<M> xo = ldg_row<M>(X, i);
      // lane l holds the entries j, j + 8, ..., of which those below j + left exist
      for (int j = j0 + l, left = cnt - l; left > 0; j += kOwnerLanes * kOwnerBatch, left -= kOwnerLanes * kOwnerBatch) {
        // the loads of kOwnerBatch entries go out before the first add; the adds keep the list order
        uint2 w[kOwnerBatch];
        float b[kOwnerBatch];
#pragma unroll
        for (int u = 0; u < kOwnerBatch; ++u) fetch(j + u * kOwnerLanes, u * kOwnerLanes < left, w[u], b[u]);
        Row<M> xn[kOwnerBatch];
#pragma unroll
        for (int u = 0; u < kOwnerBatch; ++u) xn[u] = gather(w[u], u * kOwnerLanes < left, xo);
#pragma unroll
        for (int u = 0; u < kOwnerBatch; ++u) {
          if (u * kOwnerLanes < left) {
            float v[M];
            contribution(xo, xn[u], w[u], b[u], true, v);
#pragma unroll
            for (int c = 0; c < M; ++c) acc[c] = __fadd_rn(acc[c], v[c]);
          }
        }
      }
    }
    // hubs: the whole warp evaluates 32 consecutive entries of one hub's list per round, and lane l of the hub's
    // group adds those at l, l + 8, l + 16, l + 24 -- the entries and the order of the loop above, with 4x the lanes
    // doing the math.  Two rounds ahead are in flight during a round's math and shuffles: the entry record of round
    // r + 2 and the neighbour row of round r + 1 (whose record arrived during round r - 1).
    unsigned hubs = __ballot_sync(kFull, hub && l == 0);
    while (hubs) {
      const int g0 = __ffs(hubs) - 1;  // lane 0 of the hub's group
      hubs &= hubs - 1;
      const int ih = __shfl_sync(kFull, i, g0);
      const int h0 = __shfl_sync(kFull, j0, g0), h1 = h0 + __shfl_sync(kFull, cnt, g0);
      const bool mine = (lane & ~(kOwnerLanes - 1)) == g0;
      const Row<M> xo = ldg_row<M>(X, ih);
      uint2 w0, w1;
      float b0, b1;
      fetch(h0 + lane, h0 + lane < h1, w0, b0);
      fetch(h0 + 32 + lane, h0 + 32 + lane < h1, w1, b1);
      Row<M> x0 = gather(w0, h0 + lane < h1, xo);
      for (int hb = h0; hb < h1; hb += 32) {
        const Row<M> x1 = gather(w1, hb + 32 + lane < h1, xo);
        uint2 w2;
        float b2;
        fetch(hb + 64 + lane, hb + 64 + lane < h1, w2, b2);
        float v[M];
        contribution(xo, x0, w0, b0, hb + lane < h1, v);
#pragma unroll
        for (int q = 0; q < 32 / kOwnerLanes; ++q) {
          const int from = l + q * kOwnerLanes;
#pragma unroll
          for (int c = 0; c < M; ++c) {
            const float t = __shfl_sync(kFull, v[c], from);
            if (mine && hb + from < h1) acc[c] = __fadd_rn(acc[c], t);
          }
        }
        w0 = w1; b0 = b1; x0 = x1;
        w1 = w2; b1 = b2;
      }
    }
#pragma unroll
    for (int o = kOwnerLanes / 2; o > 0; o >>= 1) {
#pragma unroll
      for (int c = 0; c < M; ++c) acc[c] += __shfl_xor_sync(kFull, acc[c], o, kOwnerLanes);
    }
    if (node && l == 0) {
#pragma unroll
      for (int c = 0; c < M; ++c) grad[(int64_t)i * M + c] += acc[c];
    }
  }
  if (MODE != 2) {
    __shared__ double sm[32];
    double v1[1] = {lsum};
    block_sum<1>(v1, sm);
    if (threadIdx.x == 0) loss_partials[blockIdx.x] = v1[0];
  }
}

// ------------------------------------------------------------------------------------------
// m >= 5: group-per-edge kernel.  G lanes share one edge; lane l owns columns l, l+G, ...
// (CPL of them).  VW = 4 treats the row as m/4 float4 columns.
// ------------------------------------------------------------------------------------------
template <int VW> struct Vec { float v[VW]; };

template <int VW>
__device__ __forceinline__ Vec<VW> ldv(const float* __restrict__ p) {
  Vec<VW> o;
  if constexpr (VW == 4) { float4 t = __ldg(reinterpret_cast<const float4*>(p)); o.v[0] = t.x; o.v[1] = t.y; o.v[2] = t.z; o.v[3] = t.w; }
  else o.v[0] = __ldg(p);
  return o;
}
template <int VW>
__device__ __forceinline__ void redv(float* p, const Vec<VW>& x, float sgn) {
  if constexpr (VW == 4) red_add_v4(p, sgn * x.v[0], sgn * x.v[1], sgn * x.v[2], sgn * x.v[3]);
  else red_add(p, sgn * x.v[0]);
}

static constexpr int kWideThreads = 256;
static constexpr int kWideSlice = 64;  // consecutive edges walked by one group

template <int G, int CPL, int VW, int MODE>
__global__ void __launch_bounds__(kWideThreads)
distortion_wide_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                       const float* __restrict__ par0, const float* __restrict__ par1,
                       const int32_t* __restrict__ perm, const float* __restrict__ gext,
                       int64_t p, int m, const float* __restrict__ X, float* __restrict__ grad,
                       double* __restrict__ loss_partials, FnDev fn, float inv_p,
                       const int* __restrict__ flag) {
  if (flag != nullptr && *flag == 0) return;
  const int lg = threadIdx.x % G;
  // shuffles stay inside the G-lane group: groups of one warp may run different trip counts
  const unsigned gmask = (G == 32) ? kFull : (((1u << G) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
  const int64_t group0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) / G;
  const int mv = m / VW;  // columns in units of VW floats
  double lsum = 0.0;

  for (int64_t k0 = group0 * kWideSlice; k0 < p; k0 += ngroups * kWideSlice) {
    int cur = -1;
    Vec<VW> xi[CPL], acc[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c)
#pragma unroll
      for (int q = 0; q < VW; ++q) { xi[c].v[q] = 0.0f; acc[c].v[q] = 0.0f; }
    // trip count is uniform across the group (shuffles inside); out-of-range iterations re-read the
    // last edge / last column (clamped indices) and are masked out of every sum and store
    for (int it = 0; it < kWideSlice; ++it) {
      const int64_t k = k0 + it;
      const bool ok = k < p;
      const int64_t kk = ok ? k : (p - 1);
      const int s = __ldg(src + kk);
      const int t = __ldg(dst + kk);
      if (ok && s != cur) {
        if (cur >= 0 && MODE != 1) {
#pragma unroll
          for (int c = 0; c < CPL; ++c) {
            int col = lg + c * G;
            if (col < mv) redv<VW>(grad + (int64_t)cur * m + col * VW, acc[c], 1.0f);
          }
        }
        cur = s;
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
          const int col = lg + c * G;
          const int colc = col < mv ? col : (mv - 1);
          xi[c] = ldv<VW>(X + (int64_t)s * m + colc * VW);
#pragma unroll
          for (int q = 0; q < VW; ++q) acc[c].v[q] = 0.0f;
        }
      }
      Vec<VW> diff[CPL];
      float d2 = 0.0f;
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        const int col = lg + c * G;
        const int colc = col < mv ? col : (mv - 1);
        const Vec<VW> xj = ldv<VW>(X + (int64_t)t * m + colc * VW);
        const float keep = (col < mv) ? 1.0f : 0.0f;
#pragma unroll
        for (int q = 0; q < VW; ++q) { diff[c].v[q] = (xi[c].v[q] - xj.v[q]) * keep; d2 += diff[c].v[q] * diff[c].v[q]; }
      }
#pragma unroll
      for (int off = G / 2; off > 0; off >>= 1) d2 += __shfl_xor_sync(gmask, d2, off);
      float g, f = 0.0f;
      if (MODE == 2) {
        g = __ldg(gext + __ldg(perm + kk));
      } else {
        const float a = __ldg(par0 + kk);
        const float b = (par1 != nullptr) ? __ldg(par1 + kk) : 1.0f;
        const float d = sqrtf(d2);
        if (MODE == 0) edge_coeff<-1, -1>(fn, d, a, b, inv_p, f, g);
        else { edge_value<-1, -1>(fn, d, a, b, f); g = 0.0f; }
        if (ok && lg == 0) lsum += (double)f;
      }
      if (MODE != 1 && ok) {
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
          int col = lg + c * G;
          if (col < mv) {
            Vec<VW> v;
#pragma unroll
            for (int q = 0; q < VW; ++q) { v.v[q] = g * diff[c].v[q]; acc[c].v[q] += v.v[q]; }
            redv<VW>(grad + (int64_t)t * m + col * VW, v, -1.0f);
          }
        }
      }
    }
    if (cur >= 0 && MODE != 1) {
#pragma unroll
      for (int c = 0; c < CPL; ++c) {
        int col = lg + c * G;
        if (col < mv) redv<VW>(grad + (int64_t)cur * m + col * VW, acc[c], 1.0f);
      }
    }
  }
  if (MODE != 2) {
    __shared__ double sm[32];
    double v1[1] = {lsum};
    block_sum<1>(v1, sm);
    if (threadIdx.x == 0) loss_partials[blockIdx.x] = v1[0];
  }
}

// ------------------------------------------------------------------------------------------
// 5 <= m <= 512, deterministic mode (MODE 0 and 2): owner-complete evaluation of the directed entries `ent`, with the
// group shape of the wide kernel.  A group of G lanes walks one owner's list in order; lane l holds columns l, l + G,
// ... of the owner row and of its gradient sum in registers.  Per entry it gathers the neighbour row, forms x_owner -
// x_neighbour, combines the squared distance over the group with a fixed xor tree and adds g (x_owner - x_neighbour).
// The lane-to-column partition and the tree are the same at both ends of an edge, and rounding is symmetric in sign,
// so both ends compute the same d, f and g.  No atomics: a row is written once, the gradient is the same bits in
// every run.  The loss counts each edge at its src-end entry, in fp64.
// Lists longer than kWideSeg entries are cut into segments of kWideSeg (the layout's `wseg` table).  The segments are
// work items of their own, evaluated in parallel into the scratch rows `wpart`; wide_owner_combine_kernel then adds
// each such node's segment rows in segment order to its gradient row.
// ------------------------------------------------------------------------------------------
static constexpr int kWideSeg = 256;

// entries per batch whose loads are issued before the first of them is added: 8 at one float of the row per lane, 4
// at 4 floats, else 2.  What stays live across the out-of-line call of the run-time function table must fit the
// registers the call preserves: at 2 floats per lane, 4 or 8 entries spill.
template <int CPL, int VW>
__host__ __device__ constexpr int wide_owner_batch() { return CPL * VW == 1 ? 8 : (CPL * VW == 4 ? 4 : 2); }

template <int G, int CPL, int VW, int MODE>
__global__ void __launch_bounds__(kWideThreads)
distortion_wide_owner_kernel(const uint2* __restrict__ ent, const uint32_t* __restrict__ inc,
                             const int64_t* __restrict__ off, const int4* __restrict__ seg, int nseg,
                             float* __restrict__ part, const float* __restrict__ par1,
                             const int32_t* __restrict__ perm, const float* __restrict__ gext, int64_t n, int m,
                             const float* __restrict__ X, float* __restrict__ grad,
                             double* __restrict__ loss_partials, FnDev fn, float inv_p,
                             const int* __restrict__ flag) {
  static_assert(MODE == 0 || MODE == 2, "value-only evaluations run on the wide kernel");
  constexpr int B = wide_owner_batch<CPL, VW>();
  if (flag != nullptr && *flag == 0) return;
  const int lg = threadIdx.x % G;
  // shuffles stay inside the G-lane group: groups of one warp walk lists of different lengths
  const unsigned gmask = (G == 32) ? kFull : (((1u << G) - 1u) << ((threadIdx.x & 31) & ~(G - 1)));
  const int64_t group0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int64_t ngroups = ((int64_t)gridDim.x * blockDim.x) / G;
  const int mv = m / VW;  // columns in units of VW floats
  const bool need_k = MODE == 2 || par1 != nullptr;
  double lsum = 0.0;
  // work items: the nseg segments of the long lists first (the largest items), then the n owners
  for (int64_t item = group0; item < nseg + n; item += ngroups) {
    int owner, jb, je;
    float* out;
    if (item < nseg) {
      const int4 s = __ldg(seg + item);
      owner = s.x; jb = s.y; je = s.z;
      out = part + item * m;
    } else {
      owner = (int)(item - nseg);
      jb = (int)ldg_stream(off + owner);
      je = (int)ldg_stream(off + owner + 1);
      if (je - jb > kWideSeg) continue;  // evaluated by its segments
      out = grad + (int64_t)owner * m;
    }
    Vec<VW> xo[CPL], acc[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      const int col = lg + c * G;
      xo[c] = ldv<VW>(X + (int64_t)owner * m + (col < mv ? col : mv - 1) * VW);
#pragma unroll
      for (int q = 0; q < VW; ++q) acc[c].v[q] = 0.0f;
    }
    // the trip count and every branch below are uniform across the group (same list)
    for (int j = jb; j < je; j += B) {
      uint2 w[B];
      float a[B], b[B];
#pragma unroll
      for (int u = 0; u < B; ++u) {
        w[u] = make_uint2(0u, 0u);
        b[u] = 1.0f;  // as the wide kernel: only WeightedQuadratic reads b, and it always has par1
        if (j + u < je) {
          w[u] = ldg_stream(ent + j + u);
          if (need_k) {
            const uint32_t k = ldg_stream(inc + j + u) >> 1;
            if (MODE == 2) w[u].y = __float_as_uint(__ldg(gext + __ldg(perm + k)));
            else b[u] = __ldg(par1 + k);
          }
        }
        a[u] = __uint_as_float(w[u].y);
      }
      Vec<VW> xn[B][CPL];
#pragma unroll
      for (int u = 0; u < B; ++u) {
        const int64_t r = (int64_t)(w[u].x & 0x7fffffffu) * m;
#pragma unroll
        for (int c = 0; c < CPL; ++c) {
          const int col = lg + c * G;
          xn[u][c] = (j + u < je) ? ldv<VW>(X + r + (col < mv ? col : mv - 1) * VW) : xo[c];
        }
      }
#pragma unroll
      for (int u = 0; u < B; ++u) {
        if (j + u < je) {
          Vec<VW> diff[CPL];
          float d2 = 0.0f;
#pragma unroll
          for (int c = 0; c < CPL; ++c) {
            const float keep = (lg + c * G < mv) ? 1.0f : 0.0f;
#pragma unroll
            for (int q = 0; q < VW; ++q) {
              diff[c].v[q] = (xo[c].v[q] - xn[u][c].v[q]) * keep;
              d2 += diff[c].v[q] * diff[c].v[q];
            }
          }
#pragma unroll
          for (int o = G / 2; o > 0; o >>= 1) d2 += __shfl_xor_sync(gmask, d2, o);
          float g;
          if (MODE == 2) {
            g = a[u];
          } else {
            float f;
            edge_coeff<-1, -1>(fn, sqrtf(d2), a[u], b[u], inv_p, f, g);
            if (lg == 0 && (w[u].x >> 31) == 0) lsum += (double)f;
          }
#pragma unroll
          for (int c = 0; c < CPL; ++c)
#pragma unroll
            for (int q = 0; q < VW; ++q) acc[c].v[q] = __fadd_rn(acc[c].v[q], __fmul_rn(g, diff[c].v[q]));
        }
      }
    }
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      const int col = lg + c * G;
      if (col < mv) {
#pragma unroll
        for (int q = 0; q < VW; ++q) {
          if (item < nseg) out[col * VW + q] = acc[c].v[q];
          else out[col * VW + q] += acc[c].v[q];
        }
      }
    }
  }
  if (MODE != 2) {
    __shared__ double sm[32];
    double v1[1] = {lsum};
    block_sum<1>(v1, sm);
    if (threadIdx.x == 0) loss_partials[blockIdx.x] = v1[0];
  }
}

// the nodes whose lists were cut into segments: grad[node] += the segment rows in segment order, one thread per
// (node, column).  whub[h] = (node, first segment, end segment).
__global__ void wide_owner_combine_kernel(const int4* __restrict__ whub, int nhub, const float* __restrict__ part,
                                          int m, float* __restrict__ grad, const int* __restrict__ flag) {
  if (flag != nullptr && *flag == 0) return;
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)nhub * m) return;
  const int h = (int)(t / m), c = (int)(t % m);
  const int4 hb = __ldg(whub + h);
  float s = __ldg(part + (int64_t)hb.y * m + c);
  for (int q = hb.y + 1; q < hb.z; ++q) s = __fadd_rn(s, __ldg(part + (int64_t)q * m + c));
  grad[(int64_t)hb.x * m + c] += s;
}

// sum of per-block partials, added to *out (single block; fixed order => deterministic)
__global__ void add_partials_kernel(const double* __restrict__ partials, int nblocks, double* out) {
  __shared__ double sm[32];
  double v[1] = {0.0};
  for (int i = threadIdx.x; i < nblocks; i += blockDim.x) v[0] += partials[i];
  block_sum<1>(v, sm);
  if (threadIdx.x == 0) out[0] += v[0];
}

// per-edge outputs in the caller's order
template <int MFIX>
__global__ void edge_outputs_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                    const float* __restrict__ par0, const float* __restrict__ par1,
                                    const int32_t* __restrict__ perm, int64_t p, int m,
                                    const float* __restrict__ X, float* __restrict__ distances,
                                    float* __restrict__ distortions, FnDev fn, const int* flag) {
  if (flag && *flag == 0) return;  // gated inside the device solver's steps (callable distortion functions)
  int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p) return;
  int s = src[k], t = dst[k];
  float d2 = 0.0f;
  for (int c = 0; c < m; ++c) {
    float df = __ldg(X + (int64_t)s * m + c) - __ldg(X + (int64_t)t * m + c);
    d2 += df * df;
  }
  float d = sqrtf(d2);
  int o = perm[k];
  if (distances) distances[o] = d;
  if (distortions) {
    float f;
    edge_value<-1, -1>(fn, d, par0[k], par1 ? par1[k] : 0.0f, f);
    distortions[o] = f;
  }
}

__global__ void function_eval_kernel(FnDev fn, const float* __restrict__ par0, int64_t par0_len,
                                     const float* __restrict__ par1, const float* __restrict__ dist,
                                     int64_t p, float* __restrict__ f_out, float* __restrict__ fp_out) {
  int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p) return;
  float a = par0[par0_len == 1 ? 0 : k];
  float b = par1 ? par1[k] : 0.0f;
  float d = dist[k];
  float f, fp;
  edge_f_fp<-1, -1>(fn, d, a, b, f, fp);
  if (f_out) f_out[k] = f;
  if (fp_out) fp_out[k] = fp;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
namespace mde {

int loss_blocks_small(int64_t p) {
  int64_t per_block = (int64_t)(kSmallThreads / 32) * 32 * kRounds;
  int64_t nb = (p + per_block - 1) / per_block;
  if (nb < 1) nb = 1;
  if (nb > kNumSMs * 8) nb = kNumSMs * 8;
  return (int)nb;
}

// A/B switches for measurements, read when a layout is created (mde_edges::kvar / nq / qbps):
//   MDE_B200_KERNEL=strided   the lane-strided kernel with the warp segmented reduction (sorted SoA)
//   MDE_B200_KERNEL=precise   the thread-contiguous / tile kernels with IEEE math instead of the MUFU forms
//   MDE_B200_NQ=2             two consecutive quads per thread in the FAST quad kernel (default 1)
//   MDE_B200_QUAD_BPS=k       blocks per SM in the quad kernel's grid cap (default 4 = one resident wave)
static void read_kernel_switches(mde_edges* e) {
  const char* ev = getenv("MDE_B200_KERNEL");
  e->kvar = 0;
  if (ev && !strcmp(ev, "strided")) e->kvar = 1;
  if (ev && !strcmp(ev, "precise")) e->kvar = 2;
  ev = getenv("MDE_B200_NQ");
  e->nq = (ev && ev[0] == '2') ? 2 : 1;
  int v = env_int("MDE_B200_QUAD_BPS", 4);
  if (v < 1) v = 1;
  if (v > 16) v = 16;
  e->qbps = v;
}

int loss_blocks_quad(int64_t p, int nq, int bps) {
  int64_t per_block = (int64_t)kQuadThreads * 4 * nq;
  int64_t nb = (p + per_block - 1) / per_block;
  if (nb < 1) nb = 1;
  if (nb > kNumSMs * bps) nb = kNumSMs * bps;
  return (int)nb;
}

// the owner kernel's grid depends on n alone; beyond kMaxLossBlocks blocks it strides over the nodes
int loss_blocks_owner(int64_t n) {
  int64_t nb = (n + kOwnerNodes - 1) / kOwnerNodes;
  if (nb < 1) nb = 1;
  if (nb > kMaxLossBlocks) nb = kMaxLossBlocks;
  return (int)nb;
}

int loss_blocks_wide(int64_t p, int G) {
  int64_t groups_per_block = kWideThreads / G;
  int64_t per_block = groups_per_block * kWideSlice;
  int64_t nb = (p + per_block - 1) / per_block;
  if (nb < 1) nb = 1;
  if (nb > kNumSMs * 8) nb = kNumSMs * 8;
  return (int)nb;
}

// compile-time function pairs of the quad / owner kernels and of the strided kernel (fused mode, m = 2 / 3)
using QuadPairs = FnList<Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG>, Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOGRATIO>, Fn1<MDE_FN_P_QUADRATIC>,
                         Fn1<MDE_FN_L_ABSOLUTE>, Fn1<MDE_FN_L_QUADRATIC>, Fn1<MDE_FN_L_WEIGHTED_QUADRATIC>,
                         Fn1<MDE_FN_L_HUBER>>;
using StridedPairs = FnList<Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG>, Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOGRATIO>,
                            Fn1<MDE_FN_P_QUADRATIC>, Fn1<MDE_FN_P_LOG1P>, Fn1<MDE_FN_L_ABSOLUTE>, Fn1<MDE_FN_L_QUADRATIC>,
                            Fn1<MDE_FN_L_WEIGHTED_QUADRATIC>, Fn1<MDE_FN_L_HUBER>>;

// one evaluation on the sorted-SoA layout; the launch helpers return the grid size (= loss partials)
struct SoaLaunch {
  const mde_edges* e;
  const float* X;
  int m;
  float* grad;
  const float* gext;
  const int* flag;
  cudaStream_t st;
  float inv_p;
  long long* fx;  // deterministic mode: the fixed-point accumulator
  bool owner;     // the owner kernel runs in place of the quad kernel
  const float* par1() const { return e->has_par1 ? e->par1 : nullptr; }
};

template <int M, int MODE, int FA, int FR, bool FAST>
int launch_owner(const SoaLaunch& l) {
  const mde_edges* e = l.e;
  const int nb = loss_blocks_owner(e->n);
  distortion_owner_kernel<M, MODE, FA, FR, FAST><<<nb, kOwnerThreads, 0, l.st>>>(
      e->ent, e->inc, e->inc_off, l.par1(), e->perm, l.gext, e->n, l.X, l.grad, e->loss_partials, e->fn, l.inv_p, l.flag);
  return nb;
}

template <int M, int MODE, int FA, int FR, bool FAST>
int launch_quad(const SoaLaunch& l) {
  if constexpr (MODE != 1) {
    if (l.owner) return launch_owner<M, MODE, FA, FR, FAST>(l);
  }
  const mde_edges* e = l.e;
  const int nq = (FAST && e->nq == 2) ? 2 : 1;
  const int nb = loss_blocks_quad(e->p, nq, e->qbps);
  auto k = nq == 2 ? &distortion_quad_kernel<M, MODE, FA, FR, FAST, 2> : &distortion_quad_kernel<M, MODE, FA, FR, FAST, 1>;
  k<<<nb, kQuadThreads, 0, l.st>>>(e->src, e->dst, e->par0, l.par1(), e->perm, l.gext, e->p, l.X, l.grad,
                                   e->loss_partials, e->fn, l.inv_p, l.flag, l.fx);
  return nb;
}

template <int M, int MODE, int FA, int FR>
int launch_strided(const SoaLaunch& l) {
  const mde_edges* e = l.e;
  const int nb = loss_blocks_small(e->p);
  distortion_small_kernel<M, MODE, FA, FR><<<nb, kSmallThreads, 0, l.st>>>(
      e->src, e->dst, e->par0, l.par1(), e->perm, l.gext, e->p, l.X, l.grad, e->loss_partials, e->fn, l.inv_p, l.flag);
  return nb;
}

template <int M, int MODE>
int launch_small(const SoaLaunch& l) {
  const FnDev& fn = l.e->fn;
  if (l.e->kvar == 1) {
    return select_fn<M, MODE>(fn, false, StridedPairs{},
                              [&](auto f) { using F = decltype(f); return launch_strided<M, MODE, F::FA, F::FR>(l); });
  }
  if constexpr (MODE == 0 && (M == 1 || M == 4)) {
    // m = 1, 4: the owner kernel evaluates every edge twice, so the recipe default PushAndPull(Log1p, Log) gets
    // compile-time ids there (IEEE math, as the run-time table) instead of two out-of-line calls
    if (l.owner && Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG>::matches(fn))
      return launch_owner<M, MODE, MDE_FN_P_LOG1P, MDE_FN_P_LOG, false>(l);
  }
  return select_fn<M, MODE>(fn, fast_log1p_log(fn, l.e->kvar == 2), QuadPairs{}, [&](auto f) {
    using F = decltype(f);
    return launch_quad<M, MODE, F::FA, F::FR, F::FAST>(l);
  });
}

// the wide owner kernel's grid depends on its work items alone (segments + owners)
int loss_blocks_wide_owner(int64_t items, int G) {
  const int64_t groups_per_block = kWideThreads / G;
  int64_t nb = (items + groups_per_block - 1) / groups_per_block;
  if (nb < 1) nb = 1;
  if (nb > kMaxLossBlocks) nb = kMaxLossBlocks;
  return (int)nb;
}

// deterministic mode at the layout's m >= 5: the owner-complete kernel, then (when some list was cut into segments)
// the kernel that adds the segment rows; both honour the step gate
template <int G, int CPL, int VW, int MODE>
int launch_wide_owner(const SoaLaunch& l) {
  const mde_edges* e = l.e;
  const int nb = loss_blocks_wide_owner(e->n + e->nwseg, G);
  distortion_wide_owner_kernel<G, CPL, VW, MODE><<<nb, kWideThreads, 0, l.st>>>(
      e->ent, e->inc, e->inc_off, e->wseg, e->nwseg, e->wpart, l.par1(), e->perm, l.gext, e->n, l.m, l.X, l.grad,
      e->loss_partials, e->fn, l.inv_p, l.flag);
  if (e->nwhub > 0) {
    ++g_launch_count;
    const int64_t t = (int64_t)e->nwhub * l.m;
    wide_owner_combine_kernel<<<ceil_div_i64(t, 256), 256, 0, l.st>>>(e->whub, e->nwhub, e->wpart, l.m, l.grad, l.flag);
  }
  return nb;
}

template <int G, int CPL, int VW, int MODE>
int launch_wide(const SoaLaunch& l) {
  const mde_edges* e = l.e;
  // the owner kernel is instantiated for the deterministic range m <= 512 (at most 16 floats of a row per lane)
  if constexpr (MODE != 1 && CPL * VW <= 16) {
    if (e->det && e->ent && l.m == e->m_hint) return launch_wide_owner<G, CPL, VW, MODE>(l);
  }
  const int nb = loss_blocks_wide(e->p, G);
  distortion_wide_kernel<G, CPL, VW, MODE><<<nb, kWideThreads, 0, l.st>>>(
      e->src, e->dst, e->par0, l.par1(), e->perm, l.gext, e->p, l.m, l.X, l.grad, e->loss_partials, e->fn, l.inv_p,
      l.flag);
  return nb;
}

template <int MODE>
int launch_distortion(const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                      int* nblocks_out, const int* flag, cudaStream_t st) {
  SoaLaunch l{e, X, m, grad, gext, flag, st, 1.0f / (float)e->p_total, nullptr, false};
  // deterministic mode (m <= 4, sorted-SoA layout): zero the fixed-point buffer, accumulate into it, add it to grad.
  // A deterministic layout built for m >= 5 has no fixed-point buffer: it evaluates its own m on the wide owner kernel
  // (launch_wide).
  if (e->det && e->fx && MODE != 1 && m <= 4 && m <= e->m_hint && e->kvar != 1) {
    l.fx = e->fx;
    const int64_t cnt = e->n * m;
    int zb = (int)((cnt + 255) / 256); if (zb > kNumSMs * 8) zb = kNumSMs * 8;
    fx_zero_kernel<<<zb, 256, 0, st>>>(flag, l.fx, cnt);
    ++g_launch_count;
  }
  // default on the sorted-SoA layout: the owner kernel over the directed entries, in place of the quad kernel
  l.owner = !l.fx && e->ent && MODE != 1 && m == e->m_hint && e->kvar != 1;
  int nb;
  if (m == 1) nb = launch_small<1, MODE>(l);
  else if (m == 2) nb = launch_small<2, MODE>(l);
  else if (m == 3) nb = launch_small<3, MODE>(l);
  else if (m == 4) nb = launch_small<4, MODE>(l);
  else if (m % 4 == 0) {
    const int mv = m / 4;
    if (mv <= 8) nb = launch_wide<8, 1, 4, MODE>(l);
    else if (mv <= 16) nb = launch_wide<16, 1, 4, MODE>(l);
    else if (mv <= 32) nb = launch_wide<32, 1, 4, MODE>(l);
    else if (mv <= 64) nb = launch_wide<32, 2, 4, MODE>(l);
    else if (mv <= 128) nb = launch_wide<32, 4, 4, MODE>(l);
    else if (mv <= 256) nb = launch_wide<32, 8, 4, MODE>(l);
    else return MDE_E_UNSUPPORTED;
  } else {
    if (m <= 8) nb = launch_wide<8, 1, 1, MODE>(l);
    else if (m <= 16) nb = launch_wide<16, 1, 1, MODE>(l);
    else if (m <= 32) nb = launch_wide<32, 1, 1, MODE>(l);
    else if (m <= 64) nb = launch_wide<32, 2, 1, MODE>(l);
    else if (m <= 128) nb = launch_wide<32, 4, 1, MODE>(l);
    else if (m <= 256) nb = launch_wide<32, 8, 1, MODE>(l);
    else if (m <= 512) nb = launch_wide<32, 16, 1, MODE>(l);
    else return MDE_E_UNSUPPORTED;
  }
  MDE_LAUNCH_CHECK();
  if (l.fx) {
    const int64_t cnt = e->n * m;
    int zb = (int)((cnt + 255) / 256); if (zb > kNumSMs * 8) zb = kNumSMs * 8;
    fx_apply_kernel<<<zb, 256, 0, st>>>(flag, l.fx, grad, cnt);
    MDE_LAUNCH_CHECK();
  }
  if (nblocks_out) *nblocks_out = nb;
  return 0;
}

int evaluate(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext, int* nblocks_out,
             const int* flag, cudaStream_t st) {
  switch (e->kind) {
    case kSoaEll:  // the fused evaluation at the layout's m; everything else on the sorted-SoA arrays
      if (mode == 0 && m == e->m_hint) return ell_launch(e, X, m, grad, nblocks_out, flag, st);
      break;
    case kPull: return pull_launch(mode, e, X, m, grad, gext, nblocks_out, flag, st);
    case kTiles: return tiled_launch(mode, e, X, m, grad, gext, nblocks_out, flag, st);
    case kSoa: break;
  }
  if (mode == 0) return launch_distortion<0>(e, X, m, grad, gext, nblocks_out, flag, st);
  if (mode == 1) return launch_distortion<1>(e, X, m, grad, gext, nblocks_out, flag, st);
  return launch_distortion<2>(e, X, m, grad, gext, nblocks_out, flag, st);
}

int edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions, const int* flag,
                 cudaStream_t st) {
  switch (e->kind) {
    case kPull: return pull_edge_outputs(e, X, m, distances, distortions, flag, st);
    case kTiles: return tiled_edge_outputs(e, X, m, distances, distortions, flag, st);
    case kSoa: case kSoaEll: break;
  }
  const int tb = 256, nb = ceil_div_i64(e->p, tb);
  edge_outputs_kernel<0><<<nb, tb, 0, st>>>(e->src, e->dst, e->par0, e->has_par1 ? e->par1 : nullptr, e->perm, e->p, m,
                                            X, distances, distortions, e->fn, flag);
  MDE_LAUNCH_CHECK();
  return 0;
}

int allow_max_smem(const void* kernel) {
  if (!kernel) return MDE_E_UNSUPPORTED;
  static std::vector<const void*> done;
  if (std::find(done.begin(), done.end(), kernel) != done.end()) return 0;
  const cudaError_t err = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDynSmem);
  if (err != cudaSuccess) return (int)err;
  done.push_back(kernel);
  return 0;
}

int split_ctas(int64_t nwt, const std::vector<int32_t>& bkt_wt0, std::vector<int32_t>& cta_wt0,
               std::vector<int32_t>& cta_bkt0) {
  const int ncta = (int)std::min<int64_t>(kNumSMs, std::max<int64_t>(1, (nwt + 1) / 2));
  cta_wt0.resize(ncta + 1);
  cta_bkt0.resize(ncta);
  for (int c = 0; c <= ncta; ++c) cta_wt0[c] = (int32_t)(nwt * c / ncta);
  for (int c = 0; c < ncta; ++c) {
    const auto it = std::upper_bound(bkt_wt0.begin(), bkt_wt0.end(), cta_wt0[c]);
    cta_bkt0[c] = (int32_t)(it - bkt_wt0.begin()) - 1;
  }
  return ncta;
}

int launch_persistent(const void* kernel, void* args, int ncta, int threads, size_t smem, int* nblocks_out,
                      cudaStream_t st) {
  const int rc = allow_max_smem(kernel);
  if (rc) return rc;
  MDE_CUDA_TRY(cudaLaunchKernel(kernel, dim3(ncta), dim3(threads), &args, smem, st));
  MDE_LAUNCH_CHECK();
  if (nblocks_out) *nblocks_out = ncta;
  return 0;
}

}  // namespace mde

extern "C" {

int mde_abi_version(void) { return MDE_ABI_VERSION; }

uint64_t mde_launch_count(void) { return (uint64_t)mde::g_launch_count; }

const char* mde_error_string(int code) {
  if (code == 0) return "ok";
  if (code > 0) return cudaGetErrorString((cudaError_t)code);
  switch (code) {
    case MDE_E_INVALID: return "mde: invalid argument";
    case MDE_E_UNSUPPORTED: return "mde: unsupported configuration";
    case MDE_E_NAN: return "mde: function or gradient evaluation returned NaN/Inf";
    case MDE_E_ALLOC: return "mde: allocation failed";
    case MDE_E_COMM: return "mde: multi-GPU handshake timed out (a peer rank never arrived)";
  }
  return "mde: unknown error";
}

int mde_edges_create(mde_edges_t** out, const int64_t* edges, int64_t p, int64_t n_items,
                     const float* par0, const float* par1, const mde_fn_t* fn, int64_t p_total,
                     void* stream) {
  return mde_edges_create_ex(out, edges, p, n_items, par0, par1, fn, p_total, 2, stream);
}

// layout choice: MDE_B200_LAYOUT=soa forces the sorted-SoA layout (quad / strided kernels), =tiles insists on
// the tile-record layout whenever it can be built; default: tiles for m <= 4 without a second parameter array
static int layout_pref() {  // read at every create: A/B runs build both layouts in one process
  const char* ev = getenv("MDE_B200_LAYOUT");
  if (ev && !strcmp(ev, "soa")) return 1;
  if (ev && !strcmp(ev, "tiles")) return 2;
  if (ev && !strcmp(ev, "pull")) return 3;
  if (ev && !strcmp(ev, "ell")) return 4;
  return 0;
}

int mde_edges_create_ex(mde_edges_t** out, const int64_t* edges, int64_t p, int64_t n_items,
                        const float* par0, const float* par1, const mde_fn_t* fn, int64_t p_total,
                        int embedding_dim, void* stream) {
  if (!out || !edges || !par0 || !fn || p <= 0 || n_items <= 0 || p >= (1ll << 31) ||
      n_items >= (1ll << 31) || p_total < p)
    return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  mde_edges* e = new (std::nothrow) mde_edges();
  if (!e) return MDE_E_ALLOC;
  e->p = p; e->n = n_items; e->p_total = p_total; e->fn = to_dev(*fn); e->has_par1 = par1 != nullptr;
  read_kernel_switches(e);

  uint64_t *keys_in = nullptr, *keys_out = nullptr;
  int32_t *vals_in = nullptr, *vals_out = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  int rc = 0, pref = 0;
  bool dense = false, want_ell = false;
#define TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { rc = (int)_e; goto fail; } } while (0)
  TRY(cudaMalloc(&e->loss_partials, sizeof(double) * kMaxLossBlocks));
  // Layout choice: the SM's L1 -> L2 request path (~1 sector request per cycle) bounds the gather / scatter; the
  // tile kernels trade requests for instructions (pull: every edge is evaluated from both ends) and win once an
  // owner's run inside a tile is long, i.e. on dense graphs (C3: 447 edges per node); on sparse ones (C2: 22, C5: 10)
  // the sorted-SoA quad kernel needs half the layout memory and no more requests per edge.
  dense = (p / n_items) >= 64;
  pref = layout_pref();
  {  // MDE_B200_DETERMINISTIC=1, sorted-SoA layout: order-independent (fixed-point) gradient accumulation for m <= 4,
     // owner-complete rows over the directed entries (built below) for 5 <= m <= 512
    const char* ev = getenv("MDE_B200_DETERMINISTIC");
    if (ev && ev[0] == '1' && embedding_dim >= 1 && embedding_dim <= 4) {
      e->det = 1; e->m_hint = embedding_dim; pref = 1;
      TRY(cudaMalloc(&e->fx, sizeof(long long) * n_items * embedding_dim));
    }
    if (ev && ev[0] == '1' && embedding_dim >= 5 && embedding_dim <= 512 && 2 * p < (1ll << 31)) {
      e->det = 1; e->m_hint = embedding_dim; pref = 1;
    }
  }
  // dense graphs: ELL pull records next to the sorted-SoA arrays (fewer instructions per entry than the flat pull
  // records) whenever the ELL builder accepts the shape (n < 2^24, <= 32 neighbour tiles);
  // MDE_B200_LAYOUT=ell asks for them on any graph
  want_ell = embedding_dim >= 1 && embedding_dim <= 4 && !par1 && !e->det && (pref == 4 || (pref == 0 && dense)) &&
             ell_supported(n_items, embedding_dim);
  if (embedding_dim >= 1 && embedding_dim <= 4 && !par1 && pref != 1 && pref != 4 && (pref != 0 || dense) && !want_ell) {
    if (pref != 2) {  // pull records
      rc = pull_build(e, edges, par0, fn, embedding_dim, st);
      if (rc == 0) { *out = e; return 0; }
      if (rc != MDE_E_UNSUPPORTED) goto fail;
    }
    if (pref != 3) {
      rc = tiled_build(e, edges, par0, fn, embedding_dim, st);
      if (rc == 0) { *out = e; return 0; }
      if (rc != MDE_E_UNSUPPORTED) goto fail;
    }
    rc = 0;  // not suited to tiles (very sparse / huge): sorted-SoA layout below
  }
  TRY(cudaMalloc(&keys_in, sizeof(uint64_t) * p));
  TRY(cudaMalloc(&keys_out, sizeof(uint64_t) * p));
  TRY(cudaMalloc(&vals_in, sizeof(int32_t) * p));
  TRY(cudaMalloc(&vals_out, sizeof(int32_t) * p));
  TRY(cudaMalloc(&e->src, sizeof(int32_t) * (p + 4)));
  TRY(cudaMalloc(&e->dst, sizeof(int32_t) * (p + 4)));
  TRY(cudaMalloc(&e->par0, sizeof(float) * (p + 4)));
  TRY(cudaMalloc(&e->perm, sizeof(int32_t) * (p + 4)));
  if (par1) TRY(cudaMalloc(&e->par1, sizeof(float) * (p + 4)));
  e->nbytes = p * (4 + 4 + 4 + 4 + (par1 ? 4 : 0)) + 8 * kMaxLossBlocks;
  {
    int tb = 256;
    int nb = ceil_div_i64(p, tb);
    make_keys_kernel<<<nb, tb, 0, st>>>(edges, par0, fn->push_pull, p, keys_in, vals_in);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p, 0, 64, st));
    TRY(cudaMalloc(&tmp, tmp_bytes));
    TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p, 0, 64, st));
    unpack_kernel<<<ceil_div_i64(p + 4, tb), tb, 0, st>>>(keys_out, vals_out, par0, par1, p, e->src, e->dst, e->par0,
                                                         e->par1, e->perm);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cudaStreamSynchronize(st));
  }
  cudaFree(keys_in); cudaFree(keys_out); cudaFree(vals_in); cudaFree(vals_out); cudaFree(tmp);
  keys_in = keys_out = nullptr; vals_in = vals_out = nullptr; tmp = nullptr;
  if (((!e->det && embedding_dim >= 1 && embedding_dim <= 4) || (e->det && embedding_dim >= 5)) && !want_ell &&
      2 * p < (1ll << 31)) {
    // incidence lists of the sorted edges: a stable radix sort by node keeps each node's entries in the order
    // (src entries by k, then dst entries by k), so the owner kernels add in the same order in every run
    uint32_t *ik = nullptr, *ik2 = nullptr, *iv = nullptr;
    int* cnt = nullptr;
    const int64_t q = 2 * p;
    size_t tb2 = 0, sb = 0;
    const int bits = bits_for((uint64_t)(n_items - 1));
    TRY(cudaMalloc(&e->ent, sizeof(uint2) * q));
    TRY(cudaMalloc(&e->inc, sizeof(uint32_t) * q));
    TRY(cudaMalloc(&e->inc_off, sizeof(int64_t) * (n_items + 1)));
    TRY(cudaMalloc(&ik, sizeof(uint32_t) * q));
    TRY(cudaMalloc(&ik2, sizeof(uint32_t) * q));
    TRY(cudaMalloc(&iv, sizeof(uint32_t) * q));
    TRY(cudaMalloc(&cnt, sizeof(int) * (n_items + 1)));
    TRY(cudaMemsetAsync(cnt, 0, sizeof(int) * (n_items + 1), st));
    inc_keys_kernel<<<ceil_div_i64(q, 256), 256, 0, st>>>(e->src, e->dst, p, ik, iv, cnt);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cub::DeviceRadixSort::SortPairs(nullptr, tb2, ik, ik2, iv, e->inc, (int)q, 0, bits, st));
    TRY(cub::DeviceScan::ExclusiveSum(nullptr, sb, cnt, e->inc_off, (int)(n_items + 1), st));
    if (sb > tb2) tb2 = sb;
    TRY(cudaMalloc(&tmp, tb2));
    TRY(cub::DeviceRadixSort::SortPairs(tmp, tb2, ik, ik2, iv, e->inc, (int)q, 0, bits, st));
    sb = tb2;
    TRY(cub::DeviceScan::ExclusiveSum(tmp, sb, cnt, e->inc_off, (int)(n_items + 1), st));
    ent_fill_kernel<<<ceil_div_i64(q, 256), 256, 0, st>>>(e->inc, e->src, e->dst, e->par0, q, e->ent);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cudaStreamSynchronize(st));
    cudaFree(ik); cudaFree(ik2); cudaFree(iv); cudaFree(cnt); cudaFree(tmp);
    tmp = nullptr;
    e->m_hint = embedding_dim;
    e->nbytes += q * 8 + q * 4 + (n_items + 1) * 8;
    if (e->det) {
      // the wide owner kernel's segments: every list longer than kWideSeg entries is cut into pieces of kWideSeg,
      // in list order; whub[h] = (node, first segment, end segment), wseg[s] = (node, first entry, end entry)
      std::vector<int64_t> off(n_items + 1);
      TRY(cudaMemcpy(off.data(), e->inc_off, sizeof(int64_t) * (n_items + 1), cudaMemcpyDeviceToHost));
      std::vector<int4> segs, hubs;
      for (int64_t i = 0; i < n_items; ++i) {
        if (off[i + 1] - off[i] <= kWideSeg) continue;
        hubs.push_back(make_int4((int)i, (int)segs.size(), 0, 0));
        for (int64_t j = off[i]; j < off[i + 1]; j += kWideSeg)
          segs.push_back(make_int4((int)i, (int)j, (int)std::min<int64_t>(j + kWideSeg, off[i + 1]), 0));
        hubs.back().z = (int)segs.size();
      }
      e->nwseg = (int)segs.size();
      e->nwhub = (int)hubs.size();
      if (e->nwhub > 0) {
        TRY(cudaMalloc(&e->wseg, sizeof(int4) * segs.size()));
        TRY(cudaMalloc(&e->whub, sizeof(int4) * hubs.size()));
        TRY(cudaMalloc(&e->wpart, sizeof(float) * segs.size() * embedding_dim));
        TRY(cudaMemcpy(e->wseg, segs.data(), sizeof(int4) * segs.size(), cudaMemcpyHostToDevice));
        TRY(cudaMemcpy(e->whub, hubs.data(), sizeof(int4) * hubs.size(), cudaMemcpyHostToDevice));
        e->nbytes += (int64_t)(segs.size() + hubs.size()) * 16 + (int64_t)segs.size() * embedding_dim * 4;
      }
    }
  }
  if (want_ell) {
    // ELL pull records next to the sorted-SoA arrays (kind 3); MDE_E_UNSUPPORTED leaves the layout at kind 0
    rc = ell_build(e, fn, embedding_dim, st);
    if (rc == (int)cudaErrorMemoryAllocation) {  // no room for the second layout: the sorted-SoA one is complete
      (void)cudaGetLastError();
      rc = MDE_E_UNSUPPORTED;
    }
    if (rc != 0 && rc != MDE_E_UNSUPPORTED) goto fail;
    rc = 0;
  }
  *out = e;
  return 0;
fail:
  cudaFree(keys_in); cudaFree(keys_out); cudaFree(vals_in); cudaFree(vals_out); cudaFree(tmp);
  mde_edges_destroy(e);
  return rc;
#undef TRY
}

int mde_edges_destroy(mde_edges_t* e) {
  if (!e) return 0;
  cudaFree(e->src); cudaFree(e->dst); cudaFree(e->perm); cudaFree(e->par0); cudaFree(e->par1);
  cudaFree(e->loss_partials); cudaFree(e->fx); cudaFree(e->ent); cudaFree(e->inc); cudaFree(e->inc_off);
  cudaFree(e->wseg); cudaFree(e->whub); cudaFree(e->wpart);
  tiled_free(e);
  pull_free(e);
  ell_free(e);
  delete e;
  return 0;
}

int64_t mde_edges_count(const mde_edges_t* e) { return e ? e->p : 0; }
int mde_edges_kind(const mde_edges_t* e) { return e ? e->kind : -1; }
int mde_edges_deterministic(const mde_edges_t* e) { return e ? e->det : 0; }
int64_t mde_edges_nbytes(const mde_edges_t* e) { return e ? e->nbytes : 0; }

int mde_distortion(const mde_edges_t* e, const float* X, int m, float* grad, double* loss_sum,
                   void* stream) {
  if (!e || !X || m < 1) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int nb = 0;
  const int rc = evaluate(grad ? 0 : 1, e, X, m, grad, nullptr, &nb, nullptr, st);
  if (rc) return rc;
  if (loss_sum) {  // NULL: leave the per-block partials (kernel-only timing)
    add_partials_kernel<<<1, 256, 0, st>>>(e->loss_partials, nb, loss_sum);
    MDE_LAUNCH_CHECK();
  }
  return 0;
}

int mde_function_eval(const mde_fn_t* fn, const float* par0, int64_t par0_len, const float* par1,
                      const float* distances, int64_t p, float* f, float* fprime, void* stream) {
  if (!fn || !par0 || !distances || p < 0 || (par0_len != 1 && par0_len != p)) return MDE_E_INVALID;
  if (p == 0) return 0;
  int tb = 256, nb = ceil_div_i64(p, tb);
  function_eval_kernel<<<nb, tb, 0, (cudaStream_t)stream>>>(to_dev(*fn), par0, par0_len, par1, distances, p, f, fprime);
  MDE_LAUNCH_CHECK();
  return 0;
}

int mde_scatter_external(const mde_edges_t* e, const float* X, int m, const float* g, float* grad,
                         void* stream) {
  if (!e || !X || !g || !grad || m < 1) return MDE_E_INVALID;
  return evaluate(2, e, X, m, grad, g, nullptr, nullptr, (cudaStream_t)stream);
}

int mde_edge_outputs(const mde_edges_t* e, const float* X, int m, float* distances, float* distortions,
                     void* stream) {
  if (!e || !X || m < 1) return MDE_E_INVALID;
  return edge_outputs(e, X, m, distances, distortions, nullptr, (cudaStream_t)stream);
}

}  // extern "C"
