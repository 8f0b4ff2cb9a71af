// mde_pull.cu -- tile-resident PULL kernel: fused average distortion (forward + backward) for m <= 4 with
// no shared-memory atomics and one global red per (owner row, neighbour tile) run.
//
// Replaces pymde/average_distortion.py:36-80.  Every undirected edge {i, j} is stored TWICE, as the directed
// entries (owner i, neighbour j) and (owner j, neighbour i); an entry contributes g (x_own - x_nbr) to the
// gradient row of its OWNER only, so the scatter-add of the reference (:77-78) becomes a sum over the sorted
// entries of an owner -- a segmented reduction in registers -- instead of two atomics per edge.
//
// Layout (mde_edges.cuh, kind 2): entries are grouped into buckets (owner super-tile, neighbour tile, class);
// a neighbour tile is R rows of X (64 KB) that one CTA keeps in shared memory, an owner super-tile keeps the
// owners' X / gradient rows L2-resident; inside a bucket entries are sorted by (owner, neighbour).  Buckets are
// padded to whole warp-tiles of 128 entries; a warp-tile is ONE contiguous 1040-byte record
//     fp32 w[128] | u16 owner - owner_base [128] | u16 neighbour - tile_base [128] | owner_base, count, class, 0
// (8.1 bytes per entry, 16.25 per undirected edge) fetched by one cp.async.bulk (TMA) into the warp's slot.
//
// A lane owns 4 consecutive entries of a warp-tile: three vector LDS fetch them, the owner rows come from global
// memory through L1 (neighbouring lanes share sectors), the neighbour rows are LDS gathers from the resident tile,
// the penalty is one-sided (a warp-tile holds one class: warp-uniform branch, 4 MUFU per entry), the run of equal
// owners is summed in registers and leaves as one vector red.  Nothing is written to shared memory after the
// tile load.
#include <cub/cub.cuh>
#include <cstring>
#include <vector>

#include "mde_edges.cuh"
#include "mde_tma.cuh"

using namespace mde;

namespace {

constexpr int kPullWarps = 32;
constexpr int kPullThreads = kPullWarps * 32;
// a warp-tile holds NE = 32 * EPL entries (EPL = entries per lane per iteration: 4 or 8); record = 2 NE + 4 words
__host__ __device__ constexpr int rec_words(int epl) { return 64 * epl + 4; }
__host__ __device__ constexpr int rec_bytes(int epl) { return rec_words(epl) * 4; }  // 1040 (EPL 4) / 2064 (EPL 8)

struct PullArgs {
  const int32_t* rec;
  const int32_t* perm;  // (edge << 1) | direction per slot, -1 for pads
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
  int x_vec_ok;
};

// 4 CONSECUTIVE entries of one lane, class known.  Entries are sorted by owner: the lane keeps the sum of a run of
// equal owners in registers (`cur`, `acc`, carried across the quads of one warp-tile) and issues one vector red when
// the owner changes, so a long run costs one red per lane that holds a piece of it.
template <int M, int MODE, int FA, int FR, bool FAST, int CLS, bool PUSH>
__device__ __forceinline__ void pull_quad(const PullArgs& a, const float* __restrict__ Xt, int ibase, int first_idx,
                                          int own_base, int cnt, const float (&w)[4], const int (&oo)[4],
                                          const int (&nl)[4], const float (&gx)[4], int& cur, float (&acc)[M],
                                          float& lsum_f, double& lsum) {
  Row<M> xi[4], xj[4];
  int own[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    own[e] = own_base + oo[e];
    xi[e] = ldg_row<M>(a.X, own[e]);
    xj[e] = lds_row<M>(Xt, nl[e]);
  }
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const bool ok = (first_idx + e) < cnt;
    float diff[M];
    float d2 = 0.0f;
#pragma unroll
    for (int c = 0; c < M; ++c) { diff[c] = xi[e].v[c] - xj[e].v[c]; d2 += diff[c] * diff[c]; }
    float g, f = 0.0f;
    if (MODE == 2) {
      g = gx[e];
    } else if (FAST) {
      edge_coeff_fast_log1p_log<CLS>(d2, w[e], a.inv_p, f, g);
    } else {
      const float d = sqrtf(d2);
      if (MODE == 0) edge_coeff<FA, FR>(a.fn, d, w[e], 0.0f, a.inv_p, f, g);
      else { edge_value<FA, FR>(a.fn, d, w[e], 0.0f, f); g = 0.0f; }
    }
    if (MODE != 2) {
      // every undirected edge is seen from both ends: count its distortion once, at the entry whose owner is
      // the smaller endpoint
      const bool canon = ok && (PUSH || own[e] < ibase + nl[e]);  // a push entry is the edge's only entry
      if (canon) { if (FAST) lsum_f += f; else lsum += (double)f; }
    }
    if (MODE != 1) {
      // d = 0: the reference replaces the non-finite g by 1 and the difference vector is 0
      const bool live = ok && (FAST ? (d2 > 0.0f) : true);
      if (own[e] != cur) {  // run ended (pads repeat the last owner: they never end one)
        red_row<M>(a.grad, cur, acc);
        cur = own[e];
#pragma unroll
        for (int c = 0; c < M; ++c) acc[c] = 0.0f;
      }
      float v[M];
#pragma unroll
      for (int c = 0; c < M; ++c) { v[c] = live ? g * diff[c] : 0.0f; acc[c] += v[c]; }
      if (PUSH && live) {  // the far endpoint of a push entry gets its contribution as one global red
        float nv[M];
#pragma unroll
        for (int c = 0; c < M; ++c) nv[c] = -v[c];
        red_row<M>(a.grad, ibase + nl[e], nv);
      }
    }
  }
}

template <int M, int MODE, int FA, int FR, bool FAST, int EPL>
__global__ void __launch_bounds__(kPullThreads, 1)
distortion_pull_kernel(const PullArgs a) {
  constexpr int NE = 32 * EPL;
  constexpr int kRecWords = rec_words(EPL), kRecBytes = rec_bytes(EPL);
  if (a.flag != nullptr && *a.flag == 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int R = 1 << a.rb;
  float* Xt = reinterpret_cast<float*>(smem_raw);
  unsigned char* slots = reinterpret_cast<unsigned char*>(Xt + R * M);
  uint64_t* bars = reinterpret_cast<uint64_t*>(slots + kPullWarps * kRecBytes);
  double* red = reinterpret_cast<double*>(bars + kPullWarps + 2);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int wt0 = __ldg(a.cta_wt0 + c), wt1 = __ldg(a.cta_wt0 + c + 1);
  int bkt = __ldg(a.cta_bkt0 + c);

  if (threadIdx.x == 0) {
#pragma unroll 1
    for (int i = 0; i <= kPullWarps; ++i) mbar_init(smem_u32(bars + i), 1);
    fence_mbar_init();
  }
  __syncthreads();

  const uint64_t pol = policy_evict_first();
  const uint32_t my_slot = smem_u32(slots + warp * kRecBytes);
  const uint32_t my_bar = smem_u32(bars + warp), x_bar = smem_u32(bars + kPullWarps);
  uint32_t ph = 0, xph = 0;

  int t = wt0 + warp;
  if (lane == 0 && t < wt1) {
    mbar_expect_tx(my_bar, kRecBytes);
    bulk_g2s_hint(my_slot, a.rec + (int64_t)t * kRecWords, kRecBytes, my_bar, pol);
  }

  int tile = -1, seg_end = wt0;
  int64_t base = 0;

  // CTA-wide: make the neighbour tile of bucket `bkt` resident.  Every warp calls it once per bucket
  // boundary of the CTA's range (same number of barriers for all warps).
  auto enter_bucket = [&]() {
    const int new_tile = __ldg(a.bkt_tile + bkt);
    const int be = __ldg(a.bkt_wt0 + bkt + 1);
    seg_end = be < wt1 ? be : wt1;
    if (new_tile == tile) return;
    __syncthreads();  // every warp is done reading the old tile
    tile = new_tile;
    base = (int64_t)tile << a.rb;
    const int64_t rows_l = a.n - base;
    const int rows = (int)(rows_l < (int64_t)R ? rows_l : (int64_t)R);
    const int nfl = rows * M;
    const float* xsrc = a.X + base * M;
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
      for (int i = (int)(bytes >> 2) + threadIdx.x; i < nfl; i += kPullThreads) Xt[i] = __ldg(xsrc + i);
      __syncthreads();
      if (bytes > 0) { mbar_wait(x_bar, xph); xph ^= 1; }
    } else {
      for (int i = threadIdx.x; i < nfl; i += kPullThreads) Xt[i] = __ldg(xsrc + i);
      __syncthreads();
    }
  };

  float lsum_f = 0.0f;
  double lsum = 0.0;
  bool first = true;

  for (; t < wt1; t += kPullWarps) {
    mbar_wait(my_bar, ph);
    ph ^= 1;
    float w[EPL];
    uint32_t op[EPL / 2], np_[EPL / 2];  // packed u16 pairs: owner offsets, neighbour rows
    int own_base, cnt, cls;
    {
      const uint32_t q = my_slot;
      asm volatile("ld.shared.s32 %0, [%1];" : "=r"(own_base) : "r"(q + 8u * NE));
      asm volatile("ld.shared.s32 %0, [%1];" : "=r"(cnt) : "r"(q + 8u * NE + 4u));
      asm volatile("ld.shared.s32 %0, [%1];" : "=r"(cls) : "r"(q + 8u * NE + 8u));
#pragma unroll
      for (int h = 0; h < EPL / 4; ++h)
        asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(w[4 * h]), "=f"(w[4 * h + 1]), "=f"(w[4 * h + 2]), "=f"(w[4 * h + 3])
                     : "r"(q + (uint32_t)(4 * EPL) * (uint32_t)lane + 16u * h));
      if constexpr (EPL == 4) {
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(op[0]), "=r"(op[1]) : "r"(q + 4u * NE + 8u * (uint32_t)lane));
        asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(np_[0]), "=r"(np_[1]) : "r"(q + 6u * NE + 8u * (uint32_t)lane));
      } else {
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(op[0]), "=r"(op[1]), "=r"(op[2]), "=r"(op[3]) : "r"(q + 4u * NE + 16u * (uint32_t)lane));
        asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(np_[0]), "=r"(np_[1]), "=r"(np_[2]), "=r"(np_[3]) : "r"(q + 6u * NE + 16u * (uint32_t)lane));
      }
    }
    // WAR on the slot: the next record may only be requested once EVERY lane's loads have returned.  A lane
    // issues the ballot only after it has consumed one element of EACH load (scoreboard wait), and the ballot
    // completes only when all lanes have issued it.  Its result guards a never-taken fence: the compiler can neither
    // drop the ballot (in every mode) nor move the refill's asm above that branch.
    {
      unsigned chk = op[EPL / 2 - 1] ^ np_[EPL / 2 - 1] ^ (unsigned)(own_base ^ cnt ^ cls);
#pragma unroll
      for (int h = 0; h < EPL / 4; ++h) chk ^= __float_as_uint(w[4 * h + 3]);  // one element of every weight load
      if (__ballot_sync(kFull, chk == 0x7fc12345u) == 0x80000001u) __threadfence_block();
    }
    if (lane == 0 && t + kPullWarps < wt1) {  // refill the slot: the record is in registers now
      mbar_expect_tx(my_bar, kRecBytes);
      bulk_g2s_hint(my_slot, a.rec + (int64_t)(t + kPullWarps) * kRecWords, kRecBytes, my_bar, pol);
    }
    while (t >= seg_end) {  // warp-uniform; CTA-wide barrier inside
      if (!first) ++bkt;
      enter_bucket();
      first = false;
    }
    float acc[M];
#pragma unroll
    for (int c = 0; c < M; ++c) acc[c] = 0.0f;
    int cur = own_base + (int)(op[0] & 0xffffu);
#pragma unroll
    for (int h = 0; h < EPL / 4; ++h) {
      const float wq[4] = {w[4 * h], w[4 * h + 1], w[4 * h + 2], w[4 * h + 3]};
      const int oq[4] = {(int)(op[2 * h] & 0xffffu), (int)(op[2 * h] >> 16), (int)(op[2 * h + 1] & 0xffffu), (int)(op[2 * h + 1] >> 16)};
      const int nq[4] = {(int)(np_[2 * h] & 0xffffu), (int)(np_[2 * h] >> 16), (int)(np_[2 * h + 1] & 0xffffu), (int)(np_[2 * h + 1] >> 16)};
      float gx[4] = {0.f, 0.f, 0.f, 0.f};
      const int first_idx = EPL * lane + 4 * h;
      if (MODE == 2) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int o = __ldg(a.perm + ((int64_t)t * NE + first_idx + e));
          gx[e] = __ldg(a.gext + (o > 0 ? (o >> 1) : 0));
        }
      }
      // class of the warp-tile (header): 0 attractive / ordinary (mirrored: pull), 1 repulsive mirrored, 2 repulsive
      // stored ONCE ("push": random pairs have no owner runs worth mirroring for)
      if (FAST) {
        if (cls == 0) pull_quad<M, MODE, FA, FR, FAST, 0, false>(a, Xt, (int)base, first_idx, own_base, cnt, wq, oq, nq, gx, cur, acc, lsum_f, lsum);
        else if (cls == 1) pull_quad<M, MODE, FA, FR, FAST, 1, false>(a, Xt, (int)base, first_idx, own_base, cnt, wq, oq, nq, gx, cur, acc, lsum_f, lsum);
        else pull_quad<M, MODE, FA, FR, FAST, 1, true>(a, Xt, (int)base, first_idx, own_base, cnt, wq, oq, nq, gx, cur, acc, lsum_f, lsum);
      } else {
        if (cls == 2) pull_quad<M, MODE, FA, FR, FAST, 2, true>(a, Xt, (int)base, first_idx, own_base, cnt, wq, oq, nq, gx, cur, acc, lsum_f, lsum);
        else pull_quad<M, MODE, FA, FR, FAST, 2, false>(a, Xt, (int)base, first_idx, own_base, cnt, wq, oq, nq, gx, cur, acc, lsum_f, lsum);
      }
    }
    if (MODE != 1 && (EPL * lane) < cnt) red_row<M>(a.grad, cur, acc);
    if (FAST) { lsum += (double)lsum_f; lsum_f = 0.0f; }
  }
  if (first && wt0 < wt1) { enter_bucket(); first = false; }
  while (seg_end < wt1) { ++bkt; enter_bucket(); }
  if (MODE != 2) {
    double v1[1] = {lsum};
    block_sum<1>(v1, red);
    if (threadIdx.x == 0) a.loss_partials[blockIdx.x] = v1[0];
  }
}

// ------------------------------------------------------------------------------------------
// layout build
// ------------------------------------------------------------------------------------------
struct PKeyBits { int rb, ss, sb, shift_own, shift_bkt; int64_t ndt; };

// entry k = (edge k >> 1, direction k & 1); key = (((owner super-tile * ndt + nbr tile) * 2 + class) | owner | nbr local)
__global__ void pull_keys_kernel(const int64_t* __restrict__ edges, const float* __restrict__ par0, int push_pull,
                                 int hybrid, uint64_t drop_bkt, int64_t p2, PKeyBits kb, uint64_t* __restrict__ keys,
                                 uint32_t* __restrict__ vals) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p2) return;
  const int64_t e = k >> 1;
  const int dir = (int)(k & 1);
  int64_t i = edges[2 * e], j = edges[2 * e + 1];
  const uint64_t cls = (push_pull && !(par0[e] >= 0.0f)) ? 1ull : 0ull;
  vals[k] = (uint32_t)k;
  if (hybrid && cls) {
    // repulsive edge stored once, owner = smaller endpoint; its mirror sorts behind every real bucket and is dropped
    if (dir) { keys[k] = drop_bkt << kb.shift_bkt; return; }
    if (i > j) { const int64_t t = i; i = j; j = t; }
  }
  const uint64_t own = (uint64_t)(dir ? j : i), nbr = (uint64_t)(dir ? i : j);
  const uint64_t bkt = (((own >> kb.ss) * (uint64_t)kb.ndt + (nbr >> kb.rb)) << 1) | cls;
  const uint64_t nl = nbr & ((1ull << kb.rb) - 1ull);
  keys[k] = (bkt << kb.shift_bkt) | (own << kb.rb) | nl;
}

__global__ void pull_starts_kernel(const uint64_t* __restrict__ keys, int64_t p2, int shift_bkt,
                                   int32_t* __restrict__ start) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p2) return;
  const uint64_t b = keys[k] >> shift_bkt;
  if (k == 0 || (keys[k - 1] >> shift_bkt) != b) start[b] = (int32_t)k;
}

__global__ void pull_fill_kernel(int32_t* __restrict__ rec, int32_t* __restrict__ perm, int64_t nwt, int epl) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < nwt * rec_words(epl)) rec[k] = 0;
  if (k < nwt * 32 * epl) perm[k] = -1;
}

// one thread per sorted entry: write its three fields; the first entry of a warp-tile also writes the header
__global__ void pull_scatter_kernel(const uint64_t* __restrict__ keys, const uint32_t* __restrict__ vals,
                                    const float* __restrict__ par0, int64_t p2, PKeyBits kb,
                                    const int32_t* __restrict__ slot_shift, const int32_t* __restrict__ grp_end,
                                    int32_t* __restrict__ rec, int32_t* __restrict__ perm, int* __restrict__ bad,
                                    int epl, int hybrid, const int32_t* __restrict__ wt_perm) {
  const int NE = 32 * epl, kRecWords = rec_words(epl);
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p2) return;
  const uint64_t key = keys[k];
  const uint64_t b = key >> kb.shift_bkt;
  const uint64_t own_mask = (1ull << kb.sb) - 1ull;
  const int32_t own = (int32_t)((key >> kb.rb) & own_mask);
  const int32_t nl = (int32_t)(key & ((1ull << kb.rb) - 1ull));
  const uint32_t v = vals[k];
  const int64_t slot = k + (int64_t)slot_shift[b];
  const int64_t t = (int64_t)wt_perm[slot / NE];  // physical position of this (logical) warp-tile
  const int j = (int)(slot % NE);
  const int64_t k0 = k - j;  // first entry of this warp-tile (same group: groups start on warp-tile boundaries)
  const int32_t own0 = (int32_t)((keys[k0] >> kb.rb) & own_mask);
  const int32_t off = own - own0;
  if (off < 0 || off > 65535) *bad = 1;
  int32_t* r = rec + t * kRecWords;
  r[j] = __float_as_int(par0[v >> 1]);
  reinterpret_cast<unsigned short*>(r + NE)[j] = (unsigned short)off;
  reinterpret_cast<unsigned short*>(r + NE + NE / 2)[j] = (unsigned short)nl;
  perm[t * NE + j] = (int32_t)v;
  if (j == 0) {
    const int64_t left = (int64_t)grp_end[b] - k0;
    const int cnt = (int)(left < NE ? left : NE);
    r[2 * NE] = own0;
    r[2 * NE + 1] = cnt;
    r[2 * NE + 2] = (b & 1ull) ? (hybrid ? 2 : 1) : 0;
    r[2 * NE + 3] = 0;
    // pads of a partial warp-tile repeat the last valid owner / neighbour so that they extend the last run
    if (cnt < NE) {
      const uint64_t kl = keys[k0 + cnt - 1];
      const unsigned short lo = (unsigned short)((int32_t)((kl >> kb.rb) & own_mask) - own0);
      const unsigned short ln = (unsigned short)(kl & ((1ull << kb.rb) - 1ull));
      for (int q = cnt; q < NE; ++q) {
        reinterpret_cast<unsigned short*>(r + NE)[q] = lo;
        reinterpret_cast<unsigned short*>(r + NE + NE / 2)[q] = ln;
      }
    }
  }
}

__global__ void pull_outputs_kernel(const int32_t* __restrict__ rec, const int32_t* __restrict__ perm,
                                    const int32_t* __restrict__ wt_tile, int rb, int epl, int64_t nslots, int m,
                                    const float* __restrict__ X, float* __restrict__ distances,
                                    float* __restrict__ distortions, FnDev fn, const int* flag) {
  if (flag && *flag == 0) return;
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nslots) return;
  const int o = perm[k];
  if (o < 0 || (o & 1)) return;  // pads, and the second direction of every edge
  const int NE = 32 * epl;
  const int64_t t = k / NE;
  const int j = (int)(k % NE);
  const int32_t* r = rec + t * rec_words(epl);
  const int s = r[2 * NE] + (int)reinterpret_cast<const unsigned short*>(r + NE)[j];
  const int d_ = (wt_tile[t] << rb) + (int)reinterpret_cast<const unsigned short*>(r + NE + NE / 2)[j];
  float d2 = 0.0f;
  for (int c = 0; c < m; ++c) {
    const float df = __ldg(X + (int64_t)s * m + c) - __ldg(X + (int64_t)d_ * m + c);
    d2 += df * df;
  }
  const float d = sqrtf(d2);
  if (distances) distances[o >> 1] = d;
  if (distortions) {
    float f;
    edge_value<-1, -1>(fn, d, __int_as_float(r[j]), 0.0f, f);
    distortions[o >> 1] = f;
  }
}

size_t pull_smem_bytes(int rb, int m, int epl) {
  return (size_t)((size_t)1 << rb) * m * sizeof(float) + (size_t)kPullWarps * rec_bytes(epl) +
         (size_t)(kPullWarps + 2) * sizeof(uint64_t) + 32 * sizeof(double);
}

// compile-time function pairs of the pull kernel
using PullPairs = FnList<Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG>, Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOGRATIO>, Fn1<MDE_FN_P_QUADRATIC>,
                         Fn1<MDE_FN_L_ABSOLUTE>, Fn1<MDE_FN_L_QUADRATIC>, Fn1<MDE_FN_L_HUBER>>;

template <int MODE>
const void* select_kernel(const mde_edges* e, int m, int epl) {
  const bool fast = fast_log1p_log(e->fn, e->precise);
  return with_small_m(m, [&](auto mc) {
    constexpr int M = decltype(mc)::value;
    return select_fn<M, MODE>(e->fn, fast, PullPairs{}, [&](auto f) {
      using F = decltype(f);
      if (epl == 8) return reinterpret_cast<const void*>(&distortion_pull_kernel<M, MODE, F::FA, F::FR, F::FAST, 8>);
      return reinterpret_cast<const void*>(&distortion_pull_kernel<M, MODE, F::FA, F::FR, F::FAST, 4>);
    });
  });
}

const void* select_kernel(const mde_edges* e, int m, int mode, int epl) {
  if (mode == 0) return select_kernel<0>(e, m, epl);
  if (mode == 1) return select_kernel<1>(e, m, epl);
  return select_kernel<2>(e, m, epl);
}

}  // namespace

namespace mde {

void pull_free(mde_edges* e) {
  cudaFree(e->wt_tile);
  e->wt_tile = nullptr;
}

// Returns 0, MDE_E_UNSUPPORTED (caller falls back to another layout) or a CUDA error.
int pull_build(mde_edges* e, const int64_t* edges, const float* par0, const mde_fn_t* fn, int m, cudaStream_t st) {
  const int64_t p = e->p, n = e->n;
  if (m < 1 || m > 4 || p >= (1ll << 30)) return MDE_E_UNSUPPORTED;
  const int64_t p2 = 2 * p;
  const int rb = tile_rb(m);
  // entries per lane per warp-tile: 8 amortises the per-record work but needs enough
  // records to keep 32 warps on every SM busy; smaller problems take 4
  int epl = (p2 / 256 >= 8ll * kPullWarps * kNumSMs) ? 8 : 4;
  { const int ev = env_int("MDE_B200_PULL_EPL", 0); if (ev == 4 || ev == 8) epl = ev; }
  const int NE = 32 * epl, kRecWords = rec_words(epl), kRecBytes = rec_bytes(epl);
  if (rb > 16 || pull_smem_bytes(rb, m, epl) > kMaxDynSmem) return MDE_E_UNSUPPORTED;
  int64_t l2_bytes = (int64_t)env_int("MDE_B200_STILE_MB", 24) << 20;  // src super-tile budget: see tiled_build
  int ss = rb;
  while (((int64_t)1 << (ss + 1)) * m * 8 <= l2_bytes && ss < 30) ++ss;
  const int64_t R = (int64_t)1 << rb, S = (int64_t)1 << ss;
  const int64_t ndt = (n + R - 1) >> rb, nst = (n + S - 1) >> ss;
  const int64_t nb_all = ndt * nst * 2;
  if (nb_all > (1ll << 22)) return MDE_E_UNSUPPORTED;
  // Hybrid (MDE_B200_PULL_REP=push; off by default): repulsive edges of PushAndPull are uniformly random pairs -- an
  // owner has ~1 of them per neighbour tile, so mirroring them doubles the work without creating runs.  Stored ONCE
  // ("push" entries: neighbour row from the shared tile, far-endpoint contribution as one global red) they cut the
  // instructions by a fifth but add one L2 request per repulsive edge for the reds, so mirroring stays the default.
  int hybrid = 0;
  { const char* ev = getenv("MDE_B200_PULL_REP"); if (ev && !strcmp(ev, "push") && fn->push_pull) hybrid = 1; }
  PKeyBits kb;
  kb.rb = rb; kb.ss = ss; kb.sb = bits_for((uint64_t)(n - 1)); kb.ndt = ndt;
  kb.shift_own = rb; kb.shift_bkt = kb.sb + rb;
  const int total_bits = kb.shift_bkt + bits_for((uint64_t)nb_all);  // bucket id nb_all = dropped mirrors
  if (total_bits > 64) return MDE_E_UNSUPPORTED;

  uint64_t *keys_in = nullptr, *keys_out = nullptr;
  uint32_t *vals_in = nullptr, *vals_out = nullptr;
  int32_t *start_d = nullptr, *shift_d = nullptr, *end_d = nullptr;
  int* bad_d = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0;
  int rc = 0;
  std::vector<int32_t> start, shift, gend, bkt_tile, bkt_wt0, cta_wt0, cta_bkt0, wt_tile, wt_perm;
  int32_t* perm_d = nullptr;
#define TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { rc = (int)_e; goto done; } } while (0)
  {
    const int tb = 256;
    const int nbk = ceil_div_i64(p2, tb);
    TRY(cudaMalloc(&keys_in, sizeof(uint64_t) * p2));
    TRY(cudaMalloc(&keys_out, sizeof(uint64_t) * p2));
    TRY(cudaMalloc(&vals_in, sizeof(uint32_t) * p2));
    TRY(cudaMalloc(&vals_out, sizeof(uint32_t) * p2));
    TRY(cudaMalloc(&start_d, sizeof(int32_t) * (nb_all + 1)));
    TRY(cudaMalloc(&shift_d, sizeof(int32_t) * nb_all));
    TRY(cudaMalloc(&end_d, sizeof(int32_t) * nb_all));
    TRY(cudaMalloc(&bad_d, sizeof(int)));
    TRY(cudaMemsetAsync(bad_d, 0, sizeof(int), st));
    pull_keys_kernel<<<nbk, tb, 0, st>>>(edges, par0, fn->push_pull, hybrid, (uint64_t)nb_all, p2, kb, keys_in, vals_in);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p2, 0, total_bits, st));
    TRY(cudaMalloc(&tmp, tmp_bytes));
    TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, keys_in, keys_out, vals_in, vals_out, (int)p2, 0, total_bits, st));
    TRY(cudaMemsetAsync(start_d, 0xFF, sizeof(int32_t) * (nb_all + 1), st));
    pull_starts_kernel<<<nbk, tb, 0, st>>>(keys_out, p2, kb.shift_bkt, start_d);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    start.resize(nb_all + 1);
    TRY(cudaMemcpyAsync(start.data(), start_d, sizeof(int32_t) * (nb_all + 1), cudaMemcpyDeviceToHost, st));
    TRY(cudaStreamSynchronize(st));
    const int64_t p2_eff = (start[nb_all] >= 0) ? (int64_t)start[nb_all] : p2;  // entries before the dropped mirrors

    shift.assign(nb_all, 0);
    gend.assign(nb_all, 0);
    // logical order: buckets (owner super-tile, neighbour tile, class) one after the other, each padded to whole
    // warp-tiles.  lb_* describe the non-empty buckets in that order.
    std::vector<int64_t> lb_id;
    std::vector<int32_t> lb_wt0;
    int64_t slot = 0, prev_b = -1;
    for (int64_t b = 0; b < nb_all; ++b) {
      if (start[b] < 0) continue;
      if (prev_b >= 0) {
        gend[prev_b] = start[b];
        const int64_t cnt = (int64_t)start[b] - (int64_t)start[prev_b];
        slot += (cnt + NE - 1) / NE * NE;
      }
      lb_id.push_back(b);
      lb_wt0.push_back((int32_t)(slot / NE));
      shift[b] = (int32_t)(slot - (int64_t)start[b]);
      prev_b = b;
    }
    if (prev_b < 0) { rc = MDE_E_INVALID; goto done; }
    gend[prev_b] = (int32_t)p2_eff;
    slot += (p2_eff - (int64_t)start[prev_b] + NE - 1) / NE * NE;
    if (slot >= (1ll << 31)) { rc = MDE_E_UNSUPPORTED; goto done; }
    const int64_t nwt = slot / NE;
    lb_wt0.push_back((int32_t)nwt);
    const int nlb = (int)lb_id.size();
    const int64_t min_per_bucket = env_int("MDE_B200_TILE_MIN", 2048);
    if (nlb > 2 && p2_eff / nlb < min_per_bucket) { rc = MDE_E_UNSUPPORTED; goto done; }
    // physical order: the two classes of one (super-tile, tile) group share the resident X tile, so their warp-tiles
    // are INTERLEAVED proportionally -- pull (issue-bound) and push (red-bound) records then alternate inside every
    // CTA instead of filling different CTAs (measured: contiguous classes left the push CTAs 3.5x longer than the rest).
    // The kernel sees one bucket per group; wt_perm maps a logical warp-tile to its physical position.
    wt_perm.assign(nwt, 0);
    for (int i0 = 0; i0 < nlb;) {
      int i1 = i0 + 1;
      if (i1 < nlb && (lb_id[i1] >> 1) == (lb_id[i0] >> 1)) ++i1;  // the group's second class
      const int32_t g0 = lb_wt0[i0], g1 = lb_wt0[i1];
      bkt_tile.push_back((int32_t)((lb_id[i0] >> 1) % ndt));
      bkt_wt0.push_back(g0);
      if (i1 - i0 == 2) {
        const int32_t nA = lb_wt0[i0 + 1] - g0, nB = g1 - lb_wt0[i0 + 1];
        int32_t ia = 0, ib = 0;
        for (int32_t t = g0; t < g1; ++t) {  // next record from the class that is behind its share
          const bool takeA = (ib >= nB) || (ia < nA && (int64_t)ia * nB <= (int64_t)ib * nA);
          if (takeA) wt_perm[g0 + ia++] = t; else wt_perm[lb_wt0[i0 + 1] + ib++] = t;
        }
      } else {
        for (int32_t t = g0; t < g1; ++t) wt_perm[t] = t;
      }
      i0 = i1;
    }
    bkt_wt0.push_back((int32_t)nwt);
    const int nbkt = (int)bkt_tile.size();

    const int ncta = split_ctas(nwt, bkt_wt0, cta_wt0, cta_bkt0);
    wt_tile.resize(nwt);
    for (int b = 0; b < nbkt; ++b)
      for (int32_t t = bkt_wt0[b]; t < bkt_wt0[b + 1]; ++t) wt_tile[t] = bkt_tile[b];

    TRY(cudaMalloc(&e->rec, sizeof(int32_t) * nwt * kRecWords));
    TRY(cudaMalloc(&e->perm, sizeof(int32_t) * nwt * NE));
    TRY(cudaMalloc(&e->bkt_tile, sizeof(int32_t) * nbkt));
    TRY(cudaMalloc(&e->bkt_wt0, sizeof(int32_t) * (nbkt + 1)));
    TRY(cudaMalloc(&e->cta_wt0, sizeof(int32_t) * (ncta + 1)));
    TRY(cudaMalloc(&e->cta_bkt0, sizeof(int32_t) * ncta));
    TRY(cudaMalloc(&e->wt_tile, sizeof(int32_t) * nwt));
    TRY(cudaMemcpyAsync(shift_d, shift.data(), sizeof(int32_t) * nb_all, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(end_d, gend.data(), sizeof(int32_t) * nb_all, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->bkt_tile, bkt_tile.data(), sizeof(int32_t) * nbkt, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->bkt_wt0, bkt_wt0.data(), sizeof(int32_t) * (nbkt + 1), cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->cta_wt0, cta_wt0.data(), sizeof(int32_t) * (ncta + 1), cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->cta_bkt0, cta_bkt0.data(), sizeof(int32_t) * ncta, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(e->wt_tile, wt_tile.data(), sizeof(int32_t) * nwt, cudaMemcpyHostToDevice, st));
    TRY(cudaMalloc(&perm_d, sizeof(int32_t) * nwt));
    TRY(cudaMemcpyAsync(perm_d, wt_perm.data(), sizeof(int32_t) * nwt, cudaMemcpyHostToDevice, st));
    pull_fill_kernel<<<ceil_div_i64(nwt * kRecWords, tb), tb, 0, st>>>(e->rec, e->perm, nwt, epl);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    pull_scatter_kernel<<<ceil_div_i64(p2_eff, tb), tb, 0, st>>>(keys_out, vals_out, par0, p2_eff, kb, shift_d, end_d, e->rec,
                                                               e->perm, bad_d, epl, hybrid, perm_d);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    int bad = 0;
    TRY(cudaMemcpyAsync(&bad, bad_d, sizeof(int), cudaMemcpyDeviceToHost, st));
    TRY(cudaStreamSynchronize(st));
    if (bad) { rc = MDE_E_UNSUPPORTED; goto done; }  // a warp-tile spans more than 65 536 owner rows (very sparse)
    e->fn = to_dev(*fn);
    for (int mode = 0; mode < 3; ++mode) {
      if ((rc = allow_max_smem(select_kernel(e, m, mode, epl)))) goto done;
    }
    e->epl = epl;
    e->kind = kPull; e->m_hint = m; e->rb = rb; e->ss = ss; e->nwt = nwt; e->nbkt = nbkt; e->ncta = ncta;
    e->nbytes = nwt * (kRecBytes + 4 * NE + 4) + 8 * kMaxLossBlocks + 4ll * (2 * nbkt + 2 * ncta + 2);
  }
done:
  cudaFree(keys_in); cudaFree(keys_out); cudaFree(vals_in); cudaFree(vals_out); cudaFree(start_d); cudaFree(shift_d);
  cudaFree(end_d); cudaFree(bad_d); cudaFree(tmp); cudaFree(perm_d);
  if (rc != 0) {
    tiled_free(e);
    pull_free(e);
    cudaFree(e->perm);
    e->perm = nullptr;
    e->kind = kSoa;
  }
  return rc;
#undef TRY
}

int pull_launch(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                int* nblocks_out, const int* flag, cudaStream_t st) {
  if (e->kind != kPull || m < 1 || m > 4) return MDE_E_UNSUPPORTED;
  const size_t smem = pull_smem_bytes(e->rb, m, e->epl);
  if (smem > kMaxDynSmem) return MDE_E_UNSUPPORTED;
  PullArgs a;
  a.rec = e->rec; a.perm = e->perm; a.gext = gext; a.bkt_tile = e->bkt_tile; a.bkt_wt0 = e->bkt_wt0;
  a.cta_wt0 = e->cta_wt0; a.cta_bkt0 = e->cta_bkt0; a.X = X; a.grad = grad; a.loss_partials = e->loss_partials;
  a.flag = flag; a.fn = e->fn; a.inv_p = 1.0f / (float)e->p_total; a.n = e->n; a.rb = e->rb;
  a.x_vec_ok = ((reinterpret_cast<uintptr_t>(X) & 15u) == 0) ? 1 : 0;
  return launch_persistent(select_kernel(e, m, mode, e->epl), &a, e->ncta, kPullThreads, smem, nblocks_out, st);
}

int pull_edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions,
                      const int* flag, cudaStream_t st) {
  const int64_t nslots = e->nwt * 32 * e->epl;
  const int tb = 256;
  pull_outputs_kernel<<<ceil_div_i64(nslots, tb), tb, 0, st>>>(e->rec, e->perm, e->wt_tile, e->rb, e->epl, nslots, m, X,
                                                              distances, distortions, e->fn, flag);
  MDE_LAUNCH_CHECK();
  return 0;
}

}  // namespace mde
