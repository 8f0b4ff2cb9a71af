// mde_tiled.cu -- tile-resident fused average-distortion kernel (forward + backward) for m <= 4.
//
// Replaces pymde/average_distortion.py:36-80 like the kernels of mde_edges.cu, with the vertex rows of one
// endpoint living in SHARED MEMORY instead of being gathered from / reduced into L2 per edge:
//
//   * layout (mde_edges.cuh, kind 1): edges grouped into buckets (src super-tile, dst tile); a dst tile is
//     R rows (R * m * 8 bytes: X tile + gradient tile, 128 KB), a src super-tile keeps its X + gradient rows
//     L2-resident; inside a bucket edges are sorted by (class, src, dst);
//   * a persistent grid of one CTA per SM walks a contiguous range of 128-edge "warp-tiles".  Every warp
//     owns a 1536-byte shared-memory slot and an mbarrier: lane 0 fetches the next record with ONE
//     cp.async.bulk (TMA, SASS UBLKCP) while the warp computes on the current one (registers are the second
//     buffer), so the 12 B/edge stream never stalls a dependent LDG;
//   * the dst tile of X arrives by cp.async.bulk too; dst-side gathers are LDS, dst-side gradient
//     contributions are shared-memory CAS adds (one 64-bit CAS per m = 2 row), the finished gradient tile is
//     flushed with coalesced 16-byte vector reds once per bucket.  The src side (sorted => runs of equal
//     src) keeps its run sum in registers and issues one global red per run, as in the quad kernel.
//
// Global L2 requests per edge drop from ~3.3 (2 row gathers + 1.3 reds) to the src side only
// (~0.2 sector reads + <= 1 red).
#include <cub/cub.cuh>
#include <vector>

#include "mde_edges.cuh"
#include "mde_tma.cuh"

using namespace mde;

namespace {

constexpr int kTileWarps = 32;                    // warps per CTA (1 CTA per SM)
constexpr int kTileThreads = kTileWarps * 32;

// (x, y) += (a, b) on an 8-byte aligned shared-memory pair: ONE 64-bit CAS per attempt (fp32 add has no native
// shared-memory atomic on sm_90a -- atomicAdd(float*) itself compiles to LDS + FADD + ATOMS.CAST.SPIN)
__device__ __forceinline__ void smem_add2(float* p, float a, float b) {
  unsigned long long* q = reinterpret_cast<unsigned long long*>(p);
  unsigned long long old = *q, assumed;
  do {
    assumed = old;
    const float lo = __uint_as_float((unsigned)(assumed & 0xffffffffull)) + a;
    const float hi = __uint_as_float((unsigned)(assumed >> 32)) + b;
    const unsigned long long nv = ((unsigned long long)__float_as_uint(hi) << 32) | (unsigned long long)__float_as_uint(lo);
    old = atomicCAS(q, assumed, nv);
  } while (old != assumed);
}

// Gt[r] -= v
template <int M>
__device__ __forceinline__ void smem_sub_row(float* __restrict__ Gt, int r, const float (&v)[M]) {
  if constexpr (M == 2) smem_add2(Gt + 2 * r, -v[0], -v[1]);
  else if constexpr (M == 4) { smem_add2(Gt + 4 * r, -v[0], -v[1]); smem_add2(Gt + 4 * r + 2, -v[2], -v[3]); }
  else {
#pragma unroll
    for (int c = 0; c < M; ++c) atomicAdd(Gt + r * M + c, -v[c]);
  }
}

struct TileArgs {
  const int32_t* rec;
  const int32_t* perm;
  const float* gext;
  const int32_t* bkt_tile;
  const int32_t* bkt_wt0;
  const int32_t* cta_wt0;
  const int32_t* cta_bkt0;
  const float* X;
  float* grad;
  double* loss_partials;
  const int* flag;
  FnDev fn;
  float inv_p;
  int64_t n;
  int rb;
  int x_vec_ok;  // X 16-byte aligned: the dst tile comes by cp.async.bulk
  int g_vec_ok;  // grad 16-byte aligned: the gradient tile is flushed with red.v4
};

// One thread, 4 consecutive slots of a warp-tile: src rows from global (L1-cached, sorted => neighbouring lanes
// share sectors), dst rows and the dst gradient in the resident tile.
template <int M, int MODE, int FA, int FR, bool FAST, int CLS>
__device__ __forceinline__ void quad_compute(const TileArgs& a, const float* __restrict__ Xt, float* __restrict__ Gt,
                                             int ibase, const int (&s)[4], const int (&td)[4], const float (&av)[4],
                                             float& lsum_f, double& lsum) {
  Row<M> xi[4], xj[4];
  int dl[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int d0 = td[e] - ibase;
    dl[e] = d0 > 0 ? d0 : 0;  // pads (dst = -1) read row 0 of the tile and are masked below
    xi[e] = ldg_row<M>(a.X, s[e]);
    xj[e] = lds_row<M>(Xt, dl[e]);
  }
  float acc[M];
#pragma unroll
  for (int cc = 0; cc < M; ++cc) acc[cc] = 0.0f;
  int cur = s[0];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const bool ok = td[e] >= 0;
    float diff[M];
    float d2 = 0.0f;
#pragma unroll
    for (int cc = 0; cc < M; ++cc) { diff[cc] = xi[e].v[cc] - xj[e].v[cc]; d2 += diff[cc] * diff[cc]; }
    float g, f = 0.0f;
    if (MODE == 2) {
      g = av[e];
    } else if (FAST) {
      edge_coeff_fast_log1p_log<CLS>(d2, av[e], a.inv_p, f, g);
    } else {
      const float d = sqrtf(d2);
      if (MODE == 0) edge_coeff<FA, FR>(a.fn, d, av[e], 0.0f, a.inv_p, f, g);
      else { edge_value<FA, FR>(a.fn, d, av[e], 0.0f, f); g = 0.0f; }
    }
    if (MODE != 2 && ok) { if (FAST) lsum_f += f; else lsum += (double)f; }
    if (MODE != 1) {
      // d = 0: the reference replaces the non-finite g by 1 and the difference vector is 0
      const bool live = ok && (FAST ? (d2 > 0.0f) : true);
      float v[M];
#pragma unroll
      for (int cc = 0; cc < M; ++cc) v[cc] = live ? g * diff[cc] : 0.0f;
      if (live) smem_sub_row<M>(Gt, dl[e], v);
      const int se = ok ? s[e] : cur;  // pads never break a run
      if (se != cur) {                 // run of equal src ended: flush its sum
        red_row<M>(a.grad, cur, acc);
        cur = se;
#pragma unroll
        for (int cc = 0; cc < M; ++cc) acc[cc] = 0.0f;
      }
#pragma unroll
      for (int cc = 0; cc < M; ++cc) acc[cc] += v[cc];
    }
  }
  if (MODE != 1) red_row<M>(a.grad, cur, acc);
  if (FAST) { lsum += (double)lsum_f; lsum_f = 0.0f; }
}

// ------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------
template <int M, int MODE, int FA, int FR, bool FAST>
__global__ void __launch_bounds__(kTileThreads, 1)
distortion_tile_kernel(const TileArgs a) {
  if (a.flag != nullptr && *a.flag == 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int R = 1 << a.rb;
  float* Xt = reinterpret_cast<float*>(smem_raw);
  float* Gt = Xt + R * M;
  unsigned char* slots = reinterpret_cast<unsigned char*>(Xt + 2 * R * M);
  uint64_t* bars = reinterpret_cast<uint64_t*>(slots + kTileWarps * kWtBytes);
  double* red = reinterpret_cast<double*>(bars + kTileWarps + 2);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int wt0 = __ldg(a.cta_wt0 + c), wt1 = __ldg(a.cta_wt0 + c + 1);
  int bkt = __ldg(a.cta_bkt0 + c);

  if (threadIdx.x == 0) {
#pragma unroll 1
    for (int i = 0; i <= kTileWarps; ++i) mbar_init(smem_u32(bars + i), 1);
    fence_mbar_init();
  }
  __syncthreads();

  const uint64_t pol = policy_evict_first();
  const uint32_t my_slot = smem_u32(slots + warp * kWtBytes);
  const uint32_t my_bar = smem_u32(bars + warp), x_bar = smem_u32(bars + kTileWarps);
  uint32_t ph = 0, xph = 0;

  int t = wt0 + warp;
  if (lane == 0 && t < wt1) {  // first record of this warp
    mbar_expect_tx(my_bar, kWtBytes);
    bulk_g2s_hint(my_slot, a.rec + (int64_t)t * kWtWords, kWtBytes, my_bar, pol);
  }

  int tile = -1, seg_end = wt0;
  int64_t base = 0;  // first row of the resident dst tile

  // CTA-wide: make the dst tile of bucket `bkt` resident (flush the finished gradient tile first).
  // Every warp calls it the same number of times (once per bucket boundary of the CTA's range).
  auto enter_bucket = [&](bool first) {
    const int new_tile = __ldg(a.bkt_tile + bkt);
    const int be = __ldg(a.bkt_wt0 + bkt + 1);
    seg_end = be < wt1 ? be : wt1;
    if (new_tile == tile) return;  // same dst tile, other src super-tile: keep accumulating
    __syncthreads();               // every warp is done with the old tile
    if (!first && MODE != 1) {
      // flush: grad[tile rows] += Gt, zero Gt (same thread reads and clears an element)
      const int64_t rows_l = a.n - base;
      const int rows = (int)(rows_l < (int64_t)R ? rows_l : (int64_t)R);
      const int nfl = rows * M;
      float* gdst = a.grad + base * M;
      if (a.g_vec_ok) {
        float4* G4 = reinterpret_cast<float4*>(Gt);
        for (int i = threadIdx.x; i < (nfl >> 2); i += kTileThreads) {
          const float4 v = G4[i];
          if (v.x != 0.0f || v.y != 0.0f || v.z != 0.0f || v.w != 0.0f) {
            red_add_v4(gdst + 4 * i, v.x, v.y, v.z, v.w);
            G4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
        for (int i = (nfl & ~3) + threadIdx.x; i < nfl; i += kTileThreads) {
          const float v = Gt[i];
          if (v != 0.0f) { red_add(gdst + i, v); Gt[i] = 0.0f; }
        }
      } else {
        for (int i = threadIdx.x; i < nfl; i += kTileThreads) {
          const float v = Gt[i];
          if (v != 0.0f) { red_add(gdst + i, v); Gt[i] = 0.0f; }
        }
      }
    }
    tile = new_tile;
    base = (int64_t)tile << a.rb;
    const int64_t rows_l = a.n - base;
    const int rows = (int)(rows_l < (int64_t)R ? rows_l : (int64_t)R);
    const int nfl = rows * M;
    const float* xsrc = a.X + base * M;
    if (first && MODE != 1) {
      float4* G4 = reinterpret_cast<float4*>(Gt);
      for (int i = threadIdx.x; i < ((R * M) >> 2); i += kTileThreads) G4[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (a.x_vec_ok) {
      const uint32_t bytes = ((uint32_t)nfl * 4u) & ~15u;
      if (threadIdx.x == 0 && bytes > 0) {
        fence_proxy_async();
        mbar_expect_tx(x_bar, bytes);
        for (uint32_t off = 0; off < bytes; off += 32768u) {
          const uint32_t chunk = (bytes - off) < 32768u ? (bytes - off) : 32768u;
          bulk_g2s(smem_u32(Xt) + off, reinterpret_cast<const unsigned char*>(xsrc) + off, chunk, x_bar);
        }
      }
      for (int i = (int)(bytes >> 2) + threadIdx.x; i < nfl; i += kTileThreads) Xt[i] = __ldg(xsrc + i);
      __syncthreads();  // zeroed / tail stores visible
      if (bytes > 0) { mbar_wait(x_bar, xph); xph ^= 1; }
    } else {
      for (int i = threadIdx.x; i < nfl; i += kTileThreads) Xt[i] = __ldg(xsrc + i);
      __syncthreads();
    }
  };

  float lsum_f = 0.0f;
  double lsum = 0.0;
  bool first = true;

  for (; t < wt1; t += kTileWarps) {
    mbar_wait(my_bar, ph);
    ph ^= 1;
    int4 s4, t4;
    float4 a4;
    {
      const uint32_t q = my_slot + (uint32_t)lane * 16u;
      asm volatile("ld.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(s4.x), "=r"(s4.y), "=r"(s4.z), "=r"(s4.w) : "r"(q));
      asm volatile("ld.shared.v4.s32 {%0, %1, %2, %3}, [%4];" : "=r"(t4.x), "=r"(t4.y), "=r"(t4.z), "=r"(t4.w) : "r"(q + 512u));
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(a4.x), "=f"(a4.y), "=f"(a4.z), "=f"(a4.w) : "r"(q + 1024u));
    }
    // WAR on the slot: the next record may only be requested once EVERY lane's loads have returned (a lane issues
    // the ballot after consuming one element of each vector load; the result guards a never-taken fence, so the
    // ballot survives in every mode and the refill's asm stays behind it)
    {
      const unsigned chk = (unsigned)(s4.w ^ t4.w) ^ __float_as_uint(a4.w);
      if (__ballot_sync(kFull, chk == 0x7fc12345u) == 0x80000001u) __threadfence_block();
    }
    if (lane == 0 && t + kTileWarps < wt1) {  // refill the slot: the record is in registers now
      mbar_expect_tx(my_bar, kWtBytes);
      bulk_g2s_hint(my_slot, a.rec + (int64_t)(t + kTileWarps) * kWtWords, kWtBytes, my_bar, pol);
    }
    while (t >= seg_end) {  // warp-uniform; CTA-wide barrier inside
      if (!first) ++bkt;
      enter_bucket(first);
      first = false;
    }

    const int s[4] = {s4.x, s4.y, s4.z, s4.w};
    const int td[4] = {t4.x, t4.y, t4.z, t4.w};
    float av[4] = {a4.x, a4.y, a4.z, a4.w};
    if (MODE == 2) {
      const int4 o4 = __ldg(reinterpret_cast<const int4*>(a.perm) + ((int64_t)t * 32 + lane));
      const int o[4] = {o4.x, o4.y, o4.z, o4.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) av[e] = __ldg(a.gext + (o[e] > 0 ? o[e] : 0));
    }
    if (FAST) {
      // edges are sorted by class inside a bucket: a warp-tile is almost always all-attractive or all-repulsive.
      // A warp-uniform branch picks the one-sided math (4 MUFU per edge instead of the 7 of the predicated
      // two-sided form); only the tile holding the class boundary takes the two-sided path.
      const bool att = (av[0] >= 0.0f) & (av[1] >= 0.0f) & (av[2] >= 0.0f) & (av[3] >= 0.0f);
      const bool rep = (av[0] < 0.0f) & (av[1] < 0.0f) & (av[2] < 0.0f) & (av[3] < 0.0f);
      if (__all_sync(kFull, att)) quad_compute<M, MODE, FA, FR, FAST, 0>(a, Xt, Gt, (int)base, s, td, av, lsum_f, lsum);
      else if (__all_sync(kFull, rep)) quad_compute<M, MODE, FA, FR, FAST, 1>(a, Xt, Gt, (int)base, s, td, av, lsum_f, lsum);
      else quad_compute<M, MODE, FA, FR, FAST, 2>(a, Xt, Gt, (int)base, s, td, av, lsum_f, lsum);
    } else {
      quad_compute<M, MODE, FA, FR, FAST, 2>(a, Xt, Gt, (int)base, s, td, av, lsum_f, lsum);
    }
  }
  // bucket boundaries this warp never reached (idle warps, short tails): take part in the CTA-wide switches
  if (first && wt0 < wt1) { enter_bucket(true); first = false; }
  while (seg_end < wt1) { ++bkt; enter_bucket(false); }
  __syncthreads();
  if (MODE != 1 && tile >= 0) {  // final flush
    const int64_t rows_l = a.n - base;
    const int rows = (int)(rows_l < (int64_t)R ? rows_l : (int64_t)R);
    const int nfl = rows * M;
    float* gdst = a.grad + base * M;
    if (a.g_vec_ok) {
      const float4* G4 = reinterpret_cast<const float4*>(Gt);
      for (int i = threadIdx.x; i < (nfl >> 2); i += kTileThreads) {
        const float4 v = G4[i];
        if (v.x != 0.0f || v.y != 0.0f || v.z != 0.0f || v.w != 0.0f) red_add_v4(gdst + 4 * i, v.x, v.y, v.z, v.w);
      }
      for (int i = (nfl & ~3) + threadIdx.x; i < nfl; i += kTileThreads) { const float v = Gt[i]; if (v != 0.0f) red_add(gdst + i, v); }
    } else {
      for (int i = threadIdx.x; i < nfl; i += kTileThreads) { const float v = Gt[i]; if (v != 0.0f) red_add(gdst + i, v); }
    }
  }
  if (MODE != 2) {
    double v1[1] = {lsum};
    block_sum<1>(v1, red);
    if (threadIdx.x == 0) a.loss_partials[blockIdx.x] = v1[0];
  }
}

// ------------------------------------------------------------------------------------------
// layout build kernels
// ------------------------------------------------------------------------------------------
struct KeyBits { int rb, ss, sb, shift_cls, shift_bkt; int64_t ndt; };

__global__ void tile_keys_kernel(const int64_t* __restrict__ edges, const float* __restrict__ par0, int push_pull,
                                 int64_t p, KeyBits kb, uint64_t* __restrict__ keys, int32_t* __restrict__ vals) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p) return;
  const int64_t i = edges[2 * k], j = edges[2 * k + 1];
  const uint64_t lo = (uint64_t)(i < j ? i : j), hi = (uint64_t)(i < j ? j : i);
  const uint64_t cls = (push_pull && !(par0[k] >= 0.0f)) ? 1ull : 0ull;
  const uint64_t bkt = (lo >> kb.ss) * (uint64_t)kb.ndt + (hi >> kb.rb);
  const uint64_t dl = hi & ((1ull << kb.rb) - 1ull);
  keys[k] = (bkt << kb.shift_bkt) | (cls << kb.shift_cls) | (lo << kb.rb) | dl;
  vals[k] = (int32_t)k;
}

__global__ void bucket_starts_kernel(const uint64_t* __restrict__ keys, int64_t p, int shift_bkt,
                                     int32_t* __restrict__ start) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p) return;
  const uint64_t b = keys[k] >> shift_bkt;
  if (k == 0 || (keys[k - 1] >> shift_bkt) != b) start[b] = (int32_t)k;
}

__global__ void fill_pads_kernel(int32_t* __restrict__ rec, int32_t* __restrict__ perm, int64_t nslots) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nslots) return;
  const int64_t t = k >> 7;
  const int j = (int)(k & 127);
  rec[t * kWtWords + j] = 0;
  rec[t * kWtWords + 128 + j] = -1;
  rec[t * kWtWords + 256 + j] = 0;
  perm[k] = -1;
}

__global__ void scatter_records_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals,
                                       const float* __restrict__ par0, int64_t p, KeyBits kb,
                                       const int32_t* __restrict__ slot_shift, int32_t* __restrict__ rec,
                                       int32_t* __restrict__ perm) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p) return;
  const uint64_t key = keys[k];
  const uint64_t b = key >> kb.shift_bkt;
  const int32_t src = (int32_t)((key >> kb.rb) & ((1ull << kb.sb) - 1ull));
  const int64_t tile = (int64_t)(b % (uint64_t)kb.ndt);
  const int32_t dst = (int32_t)((tile << kb.rb) | (int64_t)(key & ((1ull << kb.rb) - 1ull)));
  const int32_t o = vals[k];
  const int64_t slot = k + (int64_t)slot_shift[b];
  const int64_t t = slot >> 7;
  const int j = (int)(slot & 127);
  rec[t * kWtWords + j] = src;
  rec[t * kWtWords + 128 + j] = dst;
  rec[t * kWtWords + 256 + j] = __float_as_int(par0[o]);
  perm[slot] = o;
}

__global__ void tiled_outputs_kernel(const int32_t* __restrict__ rec, const int32_t* __restrict__ perm, int64_t nslots,
                                     int m, const float* __restrict__ X, float* __restrict__ distances,
                                     float* __restrict__ distortions, FnDev fn, const int* flag) {
  if (flag && *flag == 0) return;
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nslots) return;
  const int o = perm[k];
  if (o < 0) return;
  const int64_t t = k >> 7;
  const int j = (int)(k & 127);
  const int s = rec[t * kWtWords + j], d_ = rec[t * kWtWords + 128 + j];
  float d2 = 0.0f;
  for (int c = 0; c < m; ++c) {
    const float df = __ldg(X + (int64_t)s * m + c) - __ldg(X + (int64_t)d_ * m + c);
    d2 += df * df;
  }
  const float d = sqrtf(d2);
  if (distances) distances[o] = d;
  if (distortions) {
    float f;
    edge_value<-1, -1>(fn, d, __int_as_float(rec[t * kWtWords + 256 + j]), 0.0f, f);
    distortions[o] = f;
  }
}

size_t tile_smem_bytes(int rb, int m) {
  return (size_t)2 * ((size_t)1 << rb) * m * sizeof(float) + (size_t)kTileWarps * kWtBytes +
         (size_t)(kTileWarps + 2) * sizeof(uint64_t) + 32 * sizeof(double);
}

// compile-time function pairs of the tile kernel
using TilePairs = FnList<Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG>, Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOGRATIO>, Fn1<MDE_FN_P_QUADRATIC>,
                         Fn1<MDE_FN_L_ABSOLUTE>, Fn1<MDE_FN_L_QUADRATIC>, Fn1<MDE_FN_L_HUBER>>;

template <int MODE>
const void* select_kernel(const mde_edges* e, int m) {
  const bool fast = fast_log1p_log(e->fn, e->precise);
  return with_small_m(m, [&](auto mc) {
    constexpr int M = decltype(mc)::value;
    return select_fn<M, MODE>(e->fn, fast, TilePairs{}, [](auto f) {
      using F = decltype(f);
      return reinterpret_cast<const void*>(&distortion_tile_kernel<M, MODE, F::FA, F::FR, F::FAST>);
    });
  });
}

const void* select_kernel(const mde_edges* e, int m, int mode) {
  if (mode == 0) return select_kernel<0>(e, m);
  if (mode == 1) return select_kernel<1>(e, m);
  return select_kernel<2>(e, m);
}

}  // namespace

namespace mde {

void tiled_free(mde_edges* e) {
  cudaFree(e->rec); cudaFree(e->bkt_tile); cudaFree(e->bkt_wt0); cudaFree(e->cta_wt0); cudaFree(e->cta_bkt0);
  e->rec = nullptr; e->bkt_tile = e->bkt_wt0 = e->cta_wt0 = e->cta_bkt0 = nullptr;
}

// Returns 0 on success, MDE_E_UNSUPPORTED when the problem does not suit the tile layout (the caller then
// builds the sorted-SoA layout), another code on a CUDA failure.
int tiled_build(mde_edges* e, const int64_t* edges, const float* par0, const mde_fn_t* fn, int m, cudaStream_t st) {
  const int64_t p = e->p, n = e->n;
  if (m < 1 || m > 4) return MDE_E_UNSUPPORTED;
  const int rb = tile_rb(m);
  if (tile_smem_bytes(rb, m) > kMaxDynSmem) return MDE_E_UNSUPPORTED;
  // src super-tile: X + gradient rows of one super-tile (2 * m * 4 bytes per row) stay L2-resident; 24 MB leaves
  // about half of the H100's 50 MB L2 to the streamed records and the destination side
  int64_t l2_bytes = (int64_t)env_int("MDE_B200_STILE_MB", 24) << 20;
  int ss = rb;
  while (((int64_t)1 << (ss + 1)) * m * 8 <= l2_bytes && ss < 30) ++ss;
  const int64_t R = (int64_t)1 << rb, S = (int64_t)1 << ss;
  const int64_t ndt = (n + R - 1) >> rb, nst = (n + S - 1) >> ss;
  const int64_t nb_all = ndt * nst;
  if (nb_all > (1ll << 22)) return MDE_E_UNSUPPORTED;
  KeyBits kb;
  kb.rb = rb; kb.ss = ss; kb.sb = bits_for((uint64_t)(n - 1)); kb.ndt = ndt;
  kb.shift_cls = kb.sb + rb; kb.shift_bkt = kb.shift_cls + 1;
  const int total_bits = kb.shift_bkt + bits_for((uint64_t)(nb_all - 1));
  if (total_bits > 64) return MDE_E_UNSUPPORTED;

  uint64_t *keys_in = nullptr, *keys_out = nullptr;
  int32_t *vals_in = nullptr, *vals_out = nullptr, *start_d = nullptr, *shift_d = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  int rc = 0;
  std::vector<int32_t> start, shift, bkt_tile, bkt_wt0, cta_wt0, cta_bkt0;
#define TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { rc = (int)_e; goto done; } } while (0)
  {
    const int tb = 256;
    const int nbk = ceil_div_i64(p, tb);
    TRY(cudaMalloc(&keys_in, sizeof(uint64_t) * p));
    TRY(cudaMalloc(&keys_out, sizeof(uint64_t) * p));
    TRY(cudaMalloc(&vals_in, sizeof(int32_t) * p));
    TRY(cudaMalloc(&vals_out, sizeof(int32_t) * p));
    TRY(cudaMalloc(&start_d, sizeof(int32_t) * nb_all));
    TRY(cudaMalloc(&shift_d, sizeof(int32_t) * nb_all));
    tile_keys_kernel<<<nbk, tb, 0, st>>>(edges, par0, fn->push_pull, p, kb, keys_in, vals_in);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p, 0, total_bits, st));
    TRY(cudaMalloc(&tmp, tmp_bytes));
    TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p, 0, total_bits, st));
    TRY(cudaMemsetAsync(start_d, 0xFF, sizeof(int32_t) * nb_all, st));
    bucket_starts_kernel<<<nbk, tb, 0, st>>>(keys_out, p, kb.shift_bkt, start_d);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    start.resize(nb_all);
    TRY(cudaMemcpyAsync(start.data(), start_d, sizeof(int32_t) * nb_all, cudaMemcpyDeviceToHost, st));
    TRY(cudaStreamSynchronize(st));

    // host: padded bucket offsets
    shift.assign(nb_all, 0);
    int64_t slot = 0;
    int64_t prev_b = -1;
    for (int64_t b = 0; b < nb_all; ++b) {
      if (start[b] < 0) continue;
      if (prev_b >= 0) {  // close the previous bucket: its edges end where this one starts
        const int64_t cnt = (int64_t)start[b] - (int64_t)start[prev_b];
        slot += (cnt + kWtEdges - 1) / kWtEdges * kWtEdges;
      }
      bkt_tile.push_back((int32_t)(b % ndt));
      bkt_wt0.push_back((int32_t)(slot / kWtEdges));
      shift[b] = (int32_t)(slot - (int64_t)start[b]);
      prev_b = b;
    }
    if (prev_b < 0) { rc = MDE_E_INVALID; goto done; }
    {
      const int64_t cnt = p - (int64_t)start[prev_b];
      slot += (cnt + kWtEdges - 1) / kWtEdges * kWtEdges;
    }
    if (slot >= (1ll << 31)) { rc = MDE_E_UNSUPPORTED; goto done; }
    const int64_t nwt = slot / kWtEdges;
    bkt_wt0.push_back((int32_t)nwt);
    const int nbkt = (int)bkt_tile.size();
    const int64_t min_per_bucket = env_int("MDE_B200_TILE_MIN", 2048);
    if (nbkt > 1 && p / nbkt < min_per_bucket) { rc = MDE_E_UNSUPPORTED; goto done; }

    const int ncta = split_ctas(nwt, bkt_wt0, cta_wt0, cta_bkt0);

    TRY(cudaMalloc(&e->rec, sizeof(int32_t) * nwt * kWtWords));
    TRY(cudaMalloc(&e->perm, sizeof(int32_t) * nwt * kWtEdges));
    TRY(cudaMalloc(&e->bkt_tile, sizeof(int32_t) * nbkt));
    TRY(cudaMalloc(&e->bkt_wt0, sizeof(int32_t) * (nbkt + 1)));
    TRY(cudaMalloc(&e->cta_wt0, sizeof(int32_t) * (ncta + 1)));
    TRY(cudaMalloc(&e->cta_bkt0, sizeof(int32_t) * ncta));
    TRY(cudaMemcpyAsync(shift_d, shift.data(), sizeof(int32_t) * nb_all, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->bkt_tile, bkt_tile.data(), sizeof(int32_t) * nbkt, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->bkt_wt0, bkt_wt0.data(), sizeof(int32_t) * (nbkt + 1), cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->cta_wt0, cta_wt0.data(), sizeof(int32_t) * (ncta + 1), cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->cta_bkt0, cta_bkt0.data(), sizeof(int32_t) * ncta, cudaMemcpyHostToDevice, st));
    const int64_t nslots = nwt * kWtEdges;
    fill_pads_kernel<<<ceil_div_i64(nslots, tb), tb, 0, st>>>(e->rec, e->perm, nslots);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    scatter_records_kernel<<<nbk, tb, 0, st>>>(keys_out, vals_out, par0, p, kb, shift_d, e->rec, e->perm);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cudaStreamSynchronize(st));
    e->fn = to_dev(*fn);
    for (int mode = 0; mode < 3; ++mode) {
      if ((rc = allow_max_smem(select_kernel(e, m, mode)))) goto done;
    }
    e->kind = kTiles; e->m_hint = m; e->rb = rb; e->ss = ss; e->nwt = nwt; e->nbkt = nbkt; e->ncta = ncta;
    e->nbytes = nwt * (kWtBytes + 4 * kWtEdges) + 8 * kMaxLossBlocks + 4ll * (2 * nbkt + 2 * ncta + 2);
  }
done:
  cudaFree(keys_in); cudaFree(keys_out); cudaFree(vals_in); cudaFree(vals_out); cudaFree(start_d); cudaFree(shift_d);
  cudaFree(tmp);
  if (rc != 0) {
    tiled_free(e);
    cudaFree(e->perm);
    e->perm = nullptr;
    e->kind = kSoa;
  }
  return rc;
#undef TRY
}

int tiled_launch(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                 int* nblocks_out, const int* flag, cudaStream_t st) {
  if (e->kind != kTiles || m < 1 || m > 4) return MDE_E_UNSUPPORTED;
  const size_t smem = tile_smem_bytes(e->rb, m);
  if (smem > kMaxDynSmem) return MDE_E_UNSUPPORTED;  // layout built for a smaller embedding dimension
  TileArgs a;
  a.rec = e->rec; a.perm = e->perm; a.gext = gext; a.bkt_tile = e->bkt_tile; a.bkt_wt0 = e->bkt_wt0;
  a.cta_wt0 = e->cta_wt0; a.cta_bkt0 = e->cta_bkt0; a.X = X; a.grad = grad; a.loss_partials = e->loss_partials;
  a.flag = flag; a.fn = e->fn; a.inv_p = 1.0f / (float)e->p_total; a.n = e->n; a.rb = e->rb;
  a.x_vec_ok = ((reinterpret_cast<uintptr_t>(X) & 15u) == 0) ? 1 : 0;
  a.g_vec_ok = ((reinterpret_cast<uintptr_t>(grad) & 15u) == 0) ? 1 : 0;
  return launch_persistent(select_kernel(e, m, mode), &a, e->ncta, kTileThreads, smem, nblocks_out, st);
}

int tiled_edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions,
                       const int* flag, cudaStream_t st) {
  const int64_t nslots = e->nwt * kWtEdges;
  const int tb = 256;
  tiled_outputs_kernel<<<ceil_div_i64(nslots, tb), tb, 0, st>>>(e->rec, e->perm, nslots, m, X, distances, distortions,
                                                               e->fn, flag);
  MDE_LAUNCH_CHECK();
  return 0;
}

}  // namespace mde
