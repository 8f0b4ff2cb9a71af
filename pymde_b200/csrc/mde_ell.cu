// mde_ell.cu -- owner-per-lane PULL kernel ("ELL records"): fused average distortion (forward + backward) for
// m <= 4 with no atomics inside a lane, no run detection and ~half the instructions of mde_pull.cu.
//
// Replaces pymde/average_distortion.py:36-80 (gather, norm, per-edge f, mean, scatter-add).  Like mde_pull.cu every
// undirected edge {i, j} is stored as the two directed entries (owner i, neighbour j) and (owner j, neighbour i) and an
// entry only contributes to the gradient row of its OWNER.  What changes is who walks the entries:
//
//   * vertices are cut into neighbour tiles of R = 2^rb rows (64 KB of X, resident in shared memory);
//   * the entries of one (neighbour tile, class, owner) group are cut into LANE-SLOTS of at most 8 entries;
//     the lane-slots of a (tile, class) are sorted by length and packed 32 at a time into one RECORD:
//         int32 W, cls, K, nslots | u32 owner word[K][32] | K x W/2 x ( float2 w[32] | u32 neighbour pair[32] )
//     (owner word: row | count << 24 | duplicate << 31; neighbour pair: two u16 BYTE offsets of the neighbour rows
//     inside the tile; W even <= 8; K = 4 / 2 / 1 lane-slots PER LANE for W = 2 / 4 / >= 6, so that short lane-slots
//     do not pay the per-record work alone; 16 + K (128 + 192 W) bytes; column-major, so lane l reads word l of every
//     column: conflict-free).  6 bytes per directed entry = 12 bytes per edge, the size of the
//     sorted-SoA stream;
//   * ONE LANE owns one lane-slot: it loads its owner row once (LDG through L1), walks its W entries (two LDS for a
//     pair of entries + one LDS gather of the neighbour row each), keeps the gradient sum of the owner in registers
//     and leaves with ONE vector red.  No owner compare, no run flush, no u16 owner offsets, no canonical-direction
//     test (the loss is half the sum over directed entries), the trip count W is warp-uniform;
//   * pads (a lane-slot shorter than W, lanes past the last lane-slot of a group) carry w = 0 and repeat a real
//     neighbour; the generic (non-weight) functions mask them with the per-lane count instead.
//
// Records are streamed with cp.async.bulk (TMA) into two shared-memory slots per warp (mbarrier per slot, the next
// record is in flight while the current one is consumed straight from shared memory); a slot is refilled after the
// warp's last consuming instruction has issued, i.e. after every lane's LDS has returned.
//
// The layout is built on the HOST from the sorted-SoA arrays (ell_build_host: counting sorts, O(p + tiles * n)); the
// same function is exported for the CPU tests (mde_ell_host_layout), which decode the records and compare the pull
// sums with the oracle.  The sorted-SoA layout stays alongside (kind 3 = SoA + ELL): value-only evaluation, per-edge
// outputs and external coefficients run on the SoA kernels.
#include <cub/cub.cuh>
#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "mde_edges.cuh"
#include "mde_tma.cuh"

using namespace mde;

namespace {

constexpr int kEllWarps = 32;
constexpr int kEllThreads = kEllWarps * 32;
constexpr int kEllWmax = 8;                                            // entries per lane-slot
constexpr int kEllPair = 256 + 128;                                    // one column pair: float2 w[32] | u32 idx[32]
__host__ __device__ constexpr int ell_kmax(int W) { return W <= 2 ? 4 : (W <= 4 ? 2 : 1); }  // lane-slots per lane
__host__ __device__ constexpr int ell_rec_bytes(int W, int K) { return 16 + K * (128 + (W / 2) * kEllPair); }
constexpr int kEllSlotBytes = ell_rec_bytes(2, 4);                     // 2064: the largest record (W 8, K 1: 1680)
static_assert(ell_rec_bytes(4, 2) <= kEllSlotBytes && ell_rec_bytes(8, 1) <= kEllSlotBytes &&
              ell_rec_bytes(6, 1) <= kEllSlotBytes, "slot size");
constexpr uint32_t kOwnMask = 0x00ffffffu;

// Record directory: everything about the records except their bytes.  Derived from the HISTOGRAM of lane-slot lengths
// per (tile, class) alone -- lane-slots are consumed longest first inside a (tile, class) -- so the host builder and
// the device builder (which only brings that histogram back to the host) share it and produce identical layouts.
struct EllPlan {
  std::vector<uint32_t> rec_off;    // [nrec + 1], units of 16 bytes
  std::vector<int32_t> rec_hdr;     // [nrec * 4]: W, class, K, lane-slots held
  std::vector<int32_t> rec_slot0;   // [nrec] first lane-slot of the record in the globally sorted lane-slot order
  std::vector<int32_t> bkt_tile, bkt_wt0, cta_wt0, cta_bkt0;
  int ncta = 0;
  int64_t nrec = 0, nslots = 0, npadded = 0, rec_bytes = 0;
};

// hist[(tile * 2 + cls) * 9 + len]: lane-slots of length len (1..8) in (tile, cls)
int ell_plan(const uint32_t* hist, int64_t ndt, int max_cta, EllPlan& out) {
  std::vector<int64_t> rec_cost;
  out.rec_off.assign(1, 0u);
  out.rec_hdr.clear(); out.rec_slot0.clear(); out.bkt_tile.clear(); out.bkt_wt0.clear();
  out.nslots = 0; out.npadded = 0;
  int64_t bytes_total = 0, slot_base = 0;
  for (int64_t tile = 0; tile < ndt; ++tile) {
    bool tile_open = false;
    for (int64_t c = 0; c < 2; ++c) {
      const uint32_t* h = hist + (tile * 2 + c) * 9;
      int64_t total = 0;
      for (int l = 1; l <= kEllWmax; ++l) total += h[l];
      if (total == 0) continue;
      if (!tile_open) {
        out.bkt_tile.push_back((int32_t)tile);
        out.bkt_wt0.push_back((int32_t)(out.rec_off.size() - 1));
        tile_open = true;
      }
      // length of the lane-slot at position i0 of the (longest first) order
      int len = kEllWmax;
      int64_t upto = h[kEllWmax];  // lane-slots with length >= len
      for (int64_t i0 = 0; i0 < total;) {
        while (i0 >= upto) { --len; upto += h[len]; }
        const int W = (len + 1) & ~1;
        const int64_t left = total - i0;
        const int K = (int)std::min<int64_t>(ell_kmax(W), (left + 31) / 32);
        const int ns = (int)std::min<int64_t>(32ll * K, left);
        out.rec_hdr.push_back(W); out.rec_hdr.push_back((int32_t)c); out.rec_hdr.push_back(K); out.rec_hdr.push_back(ns);
        out.rec_slot0.push_back((int32_t)(slot_base + i0));
        bytes_total += ell_rec_bytes(W, K);
        out.rec_off.push_back((uint32_t)(bytes_total / 16));
        out.npadded += 32ll * K * W;
        // warp instructions (ncu source page, C2): per record, per lane-slot row, per entry column
        rec_cost.push_back(60 + (int64_t)K * (30 + (int64_t)W * (c ? 31 : 23)));
        i0 += ns;
      }
      slot_base += total;
    }
  }
  out.nslots = slot_base;
  out.nrec = (int64_t)out.rec_off.size() - 1;
  out.rec_bytes = bytes_total;
  if (out.nrec < 1 || bytes_total >= (1ll << 35) || slot_base >= (1ll << 31)) return MDE_E_UNSUPPORTED;
  out.bkt_wt0.push_back((int32_t)out.nrec);
  // persistent grid: contiguous record ranges of equal estimated cost; every tile a CTA has to load (its first one
  // and one per bucket boundary inside its range) is charged like kTileCost warp instructions
  const int ncta = (int)std::min<int64_t>(max_cta, std::max<int64_t>(1, (out.nrec + kEllWarps - 1) / kEllWarps));
  out.ncta = ncta;
  const int64_t kTileCost = 6000;
  std::vector<char> bkt_first((size_t)out.nrec, 0);
  for (size_t b = 0; b + 1 < out.bkt_wt0.size(); ++b) bkt_first[(size_t)out.bkt_wt0[b]] = 1;
  int64_t remaining = kTileCost * ((int64_t)out.bkt_tile.size() - 1 + ncta);
  for (int64_t c : rec_cost) remaining += c;
  out.cta_wt0.assign(ncta + 1, (int32_t)out.nrec);
  {
    int64_t r = 0;
    for (int c = 0; c < ncta; ++c) {
      out.cta_wt0[c] = (int32_t)r;
      if (c == ncta - 1) break;  // the last CTA takes what is left
      const int64_t budget = remaining / (ncta - c);
      int64_t acc = kTileCost;
      while (r < out.nrec) {
        const int64_t add = rec_cost[(size_t)r] + ((bkt_first[(size_t)r] && r != out.cta_wt0[c]) ? kTileCost : 0);
        if (acc + add / 2 > budget && r != out.cta_wt0[c]) break;
        acc += add;
        ++r;
      }
      remaining -= acc;
      if (remaining < 0) remaining = 0;
    }
  }
  out.cta_bkt0.resize(ncta);
  for (int c = 0; c < ncta; ++c) {
    const auto it = std::upper_bound(out.bkt_wt0.begin(), out.bkt_wt0.end(), out.cta_wt0[c]);
    int b = (int)(it - out.bkt_wt0.begin()) - 1;
    const int nb = (int)out.bkt_tile.size();
    out.cta_bkt0[c] = b < 0 ? 0 : (b >= nb ? nb - 1 : b);
  }
  return 0;
}

int ell_check_shape(int64_t n, int64_t p, int m, int rb) {
  if (m < 1 || m > 4 || n < 1 || p < 1 || n >= (1ll << 24) || p >= (1ll << 29)) return MDE_E_UNSUPPORTED;
  if (rb < 8 || rb > 15) return MDE_E_UNSUPPORTED;
  const int64_t R = 1ll << rb;
  if (((n + R - 1) >> rb) > 32) return MDE_E_UNSUPPORTED;
  if ((R - 1) * 4ll * m > 65535) return MDE_E_UNSUPPORTED;  // neighbour rows are addressed by u16 byte offsets
  return 0;
}

struct EllHost {
  std::vector<unsigned char> rec;
  EllPlan plan;
  int rb = 0;
  int64_t nentries = 0;
};

// Pure host code (CPU tests; MDE_B200_ELL_BUILD=host).  src/dst/par0: p canonical edges in any order.
int ell_build_host(int64_t n, int64_t p, int m, const int32_t* src, const int32_t* dst, const float* par0,
                   int push_pull, int rb, int max_cta, EllHost& out) {
  int rc = ell_check_shape(n, p, m, rb);
  if (rc) return rc;
  const int64_t R = 1ll << rb;
  const int64_t ndt = (n + R - 1) >> rb;
  const int64_t row_bytes = 4ll * m;
  const int64_t ng = ndt * 2 * n;  // groups (tile, class, owner)
  std::vector<uint32_t> start((size_t)ng + 1, 0u);
  auto cls_of = [&](int64_t k) -> int64_t { return (push_pull && !(par0[k] >= 0.0f)) ? 1 : 0; };
  for (int64_t k = 0; k < p; ++k) {
    const int64_t s = src[k], d = dst[k], c = cls_of(k);
    if (s < 0 || d < 0 || s >= n || d >= n) return MDE_E_INVALID;
    ++start[(size_t)((((d >> rb) * 2 + c) * n) + s) + 1];
    ++start[(size_t)((((s >> rb) * 2 + c) * n) + d) + 1];
  }
  for (int64_t g = 0; g < ng; ++g) start[(size_t)g + 1] += start[(size_t)g];
  const int64_t p2 = 2 * p;
  std::vector<float> ew((size_t)p2);
  std::vector<uint16_t> ej((size_t)p2);
  {
    std::vector<uint32_t> fill(start.begin(), start.end() - 1);
    for (int64_t k = 0; k < p; ++k) {
      const int64_t s = src[k], d = dst[k], c = cls_of(k);
      uint32_t& f1 = fill[(size_t)((((d >> rb) * 2 + c) * n) + s)];
      ew[f1] = par0[k]; ej[f1] = (uint16_t)((d & (R - 1)) * row_bytes); ++f1;
      uint32_t& f2 = fill[(size_t)((((s >> rb) * 2 + c) * n) + d)];
      ew[f2] = par0[k]; ej[f2] = (uint16_t)((s & (R - 1)) * row_bytes); ++f2;
    }
  }
  // lane-slots in (tile, class, owner, piece) order, then stably sorted by (tile, class, longest first)
  struct Slot { uint32_t first; uint32_t own; uint8_t len; };
  std::vector<Slot> sorted;
  std::vector<uint32_t> hist((size_t)ndt * 2 * 9, 0u);
  {
    std::vector<Slot> slots;
    for (int64_t tc = 0; tc < ndt * 2; ++tc) {
      slots.clear();
      for (int64_t own = 0; own < n; ++own) {
        uint32_t a = start[(size_t)(tc * n + own)];
        const uint32_t b = start[(size_t)(tc * n + own) + 1];
        while (a < b) {
          const uint32_t len = std::min<uint32_t>(kEllWmax, b - a);
          slots.push_back({a, (uint32_t)own, (uint8_t)len});
          ++hist[(size_t)tc * 9 + len];
          a += len;
        }
      }
      size_t cnt[kEllWmax + 2] = {0};
      for (const Slot& sl : slots) ++cnt[kEllWmax - sl.len + 1];
      for (int i = 0; i <= kEllWmax; ++i) cnt[i + 1] += cnt[i];
      const size_t base = sorted.size();
      sorted.resize(base + slots.size());
      for (const Slot& sl : slots) sorted[base + cnt[kEllWmax - sl.len]++] = sl;
    }
  }
  rc = ell_plan(hist.data(), ndt, max_cta, out.plan);
  if (rc) return rc;
  const EllPlan& pl = out.plan;
  out.rb = rb; out.nentries = p2;
  out.rec.assign((size_t)pl.rec_bytes, 0);
  for (int64_t t = 0; t < pl.nrec; ++t) {
    const int W = pl.rec_hdr[4 * t], K = pl.rec_hdr[4 * t + 2], ns = pl.rec_hdr[4 * t + 3];
    unsigned char* r = out.rec.data() + ((size_t)pl.rec_off[(size_t)t] << 4);
    memcpy(r, &pl.rec_hdr[4 * t], 16);
    uint32_t* ow = reinterpret_cast<uint32_t*>(r + 16);
    unsigned char* cols = r + 16 + 128 * K;
    const size_t i0 = (size_t)pl.rec_slot0[(size_t)t];
    for (int i = 0; i < 32 * K; ++i) {
      const int k = i / 32, l = i % 32;
      const bool dup = i >= ns;
      const Slot& sl = sorted[i0 + (dup ? 0 : i)];
      ow[i] = sl.own | (dup ? 0x80000000u : ((uint32_t)sl.len << 24));
      unsigned char* cb = cols + (size_t)k * (W / 2) * kEllPair;
      for (int e = 0; e < W; ++e) {
        const bool real = !dup && e < (int)sl.len;
        const uint32_t src_e = sl.first + (uint32_t)std::min<int>(e, (int)sl.len - 1);
        float* wp = reinterpret_cast<float*>(cb + (e / 2) * kEllPair) + 2 * l + (e & 1);
        uint16_t* ip = reinterpret_cast<uint16_t*>(cb + (e / 2) * kEllPair + 256) + 2 * l + (e & 1);
        *wp = real ? ew[src_e] : 0.0f;
        *ip = ej[src_e];
      }
    }
  }
  return 0;
}

// ------------------------------------------------------------------------------------------
// kernel
// ------------------------------------------------------------------------------------------
struct EllArgs {
  const unsigned char* rec;
  const uint32_t* rec_off;
  const int32_t* bkt_tile;
  const int32_t* bkt_wt0;
  const int4* cta_desc;  // per CTA: first record, end record, first bucket, neighbour tile of that bucket
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

// PushAndPull(Log1p(1.5), Log(1.0)), MUFU math, class known at compile time.  Same formulas as
// mde_common.cuh::edge_coeff_fast_log1p_log; returns the loss in log2 units (flog2 = w lg2(.), the block sum is
// multiplied by ln 2 at the end) and gs = f'/(p d) WITHOUT the class constant (1.5/p attractive, 1/p repulsive: applied
// once per lane-slot to the accumulated row); gs = 0 at d = 0 (the reference replaces the non-finite g, and the
// difference vector is 0).
template <int CLS>
__device__ __forceinline__ void ell_fast_coeff(float d2, float w, float& flog2, float& gs) {
  const float kLog2e = 1.44269504089f;
  if constexpr (CLS == 0) {
    // d2 = 0: rsqrt of the clamp is finite, d = 0 * finite = 0, sqrt(0) = 0 -> gs = 0 without a select
    const float rs = fast_rsqrt(fmaxf(d2, 1e-30f));
    const float d = d2 * rs;
    const float sd = fast_sqrt(d);
    const float one_p = fmaf(d, sd, 1.0f);
    flog2 = w * fast_lg2(one_p);
    gs = (sd * rs) * fast_rcp(one_p) * w;
  } else {
    const float rs = fast_rsqrt(d2);
    const bool pos = d2 > 0.0f;
    const float d = pos ? d2 * rs : 0.0f;
    const float em = fast_ex2(-d * kLog2e);
    float one_m = 1.0f - em;
    const float series = d * (1.0f - d * (0.5f - d * (0.16666667f - d * 0.041666668f)));
    one_m = (d < 0.0625f) ? series : one_m;
    flog2 = w * fast_lg2(one_m);
    const float gg = (rs * em) * fast_rcp(one_m) * w;
    gs = pos ? gg : 0.0f;
  }
}

// f' of these functions is finite at d = 0, so g = f'/(p d) can be formed from a clamped rsqrt without any guard
// (at d = 0 the difference vector is 0 and a finite g contributes nothing, like the reference's replacement value)
template <int FA, int FR>
struct EllFiniteAtZero {
  static constexpr bool value = (FA == FR) && (FA == MDE_FN_L_HUBER || FA == MDE_FN_L_QUADRATIC || FA == MDE_FN_P_QUADRATIC);
};

// MASK: the lane-slot row has pads (entries e >= cnt) that the generic functions must not see; rows whose 32 lane-slots
// all hold W entries (almost all of them: lane-slots are sorted by length) run without the two selects
template <int M, int FA, int FR, bool FAST, int CLS, bool MASK>
__device__ __forceinline__ void ell_entry(const EllArgs& a, const float* __restrict__ Xt, const Row<M>& xi, float w,
                                          uint32_t j, bool valid, float (&acc)[M], float& lf) {
  float xj[M], diff[M];
  lds_row_at<M>(Xt, j, xj);
  float d2 = 0.0f;
#pragma unroll
  for (int c = 0; c < M; ++c) { diff[c] = xi.v[c] - xj[c]; d2 = fmaf(diff[c], diff[c], d2); }
  float f, g;
  if constexpr (FAST) {
    ell_fast_coeff<CLS>(d2, w, f, g);  // pads: w = 0
  } else {
    // d and 1/d from ONE rsqrt.approx (<= 2 ulp) instead of an IEEE sqrt and an IEEE division (18 instructions)
    float fp;
    if constexpr (EllFiniteAtZero<FA, FR>::value) {
      const float rs = fast_rsqrt(fmaxf(d2, 1e-30f));
      const float d = d2 * rs;
      edge_f_fp<FA, FR>(a.fn, d, w, 0.0f, f, fp);
      g = (fp * a.inv_p) * rs;
    } else {
      // d = 0: g is non-finite -> 1 like the reference (average_distortion.py:55-62), the difference vector is 0
      const float rs = fast_rsqrt(d2);
      const float d = (d2 > 0.0f) ? d2 * rs : 0.0f;
      edge_f_fp<FA, FR>(a.fn, d, w, 0.0f, f, fp);
      g = (fp * a.inv_p) * rs;
      if (!isfinite(g)) g = 1.0f;
    }
    if constexpr (MASK) {
      f = valid ? f : 0.0f;
      g = valid ? g : 0.0f;
    }
  }
  lf += f;
#pragma unroll
  for (int c = 0; c < M; ++c) acc[c] = fmaf(g, diff[c], acc[c]);
}

// all W entries of this lane's lane-slot, straight from the shared-memory slot
template <int M, int FA, int FR, bool FAST, int CLS, bool MASK>
__device__ __forceinline__ void ell_columns(const EllArgs& a, const float* __restrict__ Xt, const unsigned char* cols,
                                            int lane, int W, int cnt, const Row<M>& xi, float (&acc)[M],
                                            float& lf) {
  const float2* wp = reinterpret_cast<const float2*>(cols) + lane;
  const uint32_t* ip = reinterpret_cast<const uint32_t*>(cols + 256) + lane;
#pragma unroll 2
  for (int c2 = 0; 2 * c2 < W; ++c2) {
    const float2 w2 = wp[c2 * (kEllPair / 8)];
    const uint32_t ix = ip[c2 * (kEllPair / 4)];
    ell_entry<M, FA, FR, FAST, CLS, MASK>(a, Xt, xi, w2.x, ix & 0xffffu, 2 * c2 < cnt, acc, lf);
    ell_entry<M, FA, FR, FAST, CLS, MASK>(a, Xt, xi, w2.y, ix >> 16, 2 * c2 + 1 < cnt, acc, lf);
  }
}

template <int M, int FA, int FR, bool FAST>
__global__ void __launch_bounds__(kEllThreads, 1)
distortion_ell_kernel(const EllArgs a) {
  if (a.flag != nullptr && *a.flag == 0) return;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int R = 1 << a.rb;
  float* Xt = reinterpret_cast<float*>(smem_raw);
  unsigned char* slots = reinterpret_cast<unsigned char*>(Xt + R * M);
  uint64_t* bars = reinterpret_cast<uint64_t*>(slots + 2 * kEllWarps * kEllSlotBytes);
  double* red = reinterpret_cast<double*>(bars + 2 * kEllWarps + 2);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x;
  const int4 dsc = __ldg(a.cta_desc + c);  // ONE dependent load before the first copies can be issued
  const int wt0 = dsc.x, wt1 = dsc.y;
  int bkt = dsc.z;

  if (threadIdx.x == 0) {
#pragma unroll 1
    for (int i = 0; i <= 2 * kEllWarps; ++i) mbar_init(smem_u32(bars + i), 1);
    fence_mbar_init();
  }
  __syncthreads();

  const uint64_t pol = policy_evict_first();
  unsigned char* my_slots = slots + (size_t)warp * 2 * kEllSlotBytes;
  const uint32_t my_slot0 = smem_u32(my_slots);
  const uint32_t my_bar0 = smem_u32(bars + 2 * warp), x_bar = smem_u32(bars + 2 * kEllWarps);
  uint32_t phbits = 0, xph = 0;

  // lane 0 streams this warp's records (wt0 + warp, + 32, ...) two deep
  auto issue = [&](uint32_t o0, uint32_t o1, int s) {
    const uint32_t bytes = (o1 - o0) << 4;
    const uint32_t bar = my_bar0 + 8u * (uint32_t)s;
    mbar_expect_tx(bar, bytes);
    bulk_g2s_hint(my_slot0 + (uint32_t)s * kEllSlotBytes, a.rec + ((size_t)o0 << 4), bytes, bar, pol);
  };
  int tile = -1, seg_end = wt0;
  bool tile_pending = false;

  // CTA-wide: request neighbour tile `tl` (thread 0: bulk copies; everybody: the unaligned tail) / wait for it
  auto tile_issue = [&](int tl) {
    tile = tl;
    const int64_t base = (int64_t)tile << a.rb;
    const int64_t rows_l = a.n - base;
    const int rows = (int)(rows_l < (int64_t)R ? rows_l : (int64_t)R);
    const int nfl = rows * M;
    const float* xsrc = a.X + base * M;
    const uint32_t bytes = a.x_vec_ok ? (((uint32_t)nfl * 4u) & ~15u) : 0u;
    if (threadIdx.x == 0 && bytes > 0) {
      fence_proxy_async();
      mbar_expect_tx(x_bar, bytes);
      for (uint32_t off = 0; off < bytes; off += 32768u) {
        const uint32_t chunk = (bytes - off) < 32768u ? (bytes - off) : 32768u;
        bulk_g2s(smem_u32(Xt) + off, reinterpret_cast<const unsigned char*>(xsrc) + off, chunk, x_bar);
      }
    }
    for (int i = (int)(bytes >> 2) + threadIdx.x; i < nfl; i += kEllThreads) Xt[i] = __ldg(xsrc + i);
    tile_pending = true;
    return bytes;
  };
  uint32_t tile_bytes = 0;
  auto tile_wait = [&]() {
    __syncthreads();  // the plain-load tail of every thread
    if (tile_bytes > 0) { mbar_wait(x_bar, xph); xph ^= 1; }
    tile_pending = false;
  };
  // the tile of the first bucket is requested NOW: its copy overlaps the record-offset loads and the first record copies
  if (wt0 < wt1) tile_bytes = tile_issue(dsc.w);

  int t = wt0 + warp;
  if (lane == 0) {
    if (t < wt1) issue(__ldg(a.rec_off + t), __ldg(a.rec_off + t + 1), 0);
    if (t + kEllWarps < wt1) issue(__ldg(a.rec_off + t + kEllWarps), __ldg(a.rec_off + t + kEllWarps + 1), 1);
  }

  // make the neighbour tile of bucket `bkt` resident (same number of barriers for all warps)
  auto enter_bucket = [&]() {
    const int new_tile = __ldg(a.bkt_tile + bkt);
    const int be = __ldg(a.bkt_wt0 + bkt + 1);
    seg_end = be < wt1 ? be : wt1;
    if (new_tile != tile) {
      __syncthreads();  // every warp is done reading the old tile
      tile_bytes = tile_issue(new_tile);
    }
    if (tile_pending) tile_wait();
  };

  const float c_att = 1.5f * a.inv_p;
  double lsum = 0.0;
  bool first = true;
  int s = 0;

  for (; t < wt1; t += kEllWarps, s ^= 1) {
    // offsets of the record that will re-fill this slot (two records ahead): requested now, needed after the columns
    const int t2 = t + 2 * kEllWarps;
    uint32_t o0 = 0, o1 = 0;
    if (lane == 0 && t2 < wt1) { o0 = __ldg(a.rec_off + t2); o1 = __ldg(a.rec_off + t2 + 1); }
    // bucket change first: at the start of the kernel the tile copy then overlaps the first record copies
    while (t >= seg_end) {  // warp-uniform; CTA-wide barrier inside
      if (!first) ++bkt;
      enter_bucket();
      first = false;
    }
    mbar_wait(my_bar0 + 8u * (uint32_t)s, (phbits >> s) & 1u);
    phbits ^= 1u << s;
    const unsigned char* rec = my_slots + (size_t)s * kEllSlotBytes;
    const int4 hdr = *reinterpret_cast<const int4*>(rec);  // W, class, K, nslots (broadcast)
    const int W = hdr.x, K = hdr.z;
    const unsigned char* cols = rec + 16 + 128 * K;
    const int row_bytes = (W >> 1) * kEllPair;
    float lrec = 0.0f;
#pragma unroll 1
    for (int k = 0; k < K; ++k) {  // K lane-slots per lane (warp-uniform)
      const uint32_t ow = reinterpret_cast<const uint32_t*>(rec + 16)[k * 32 + lane];
      const uint32_t own = ow & kOwnMask;
      const int cnt = (int)((ow >> 24) & 0x7fu);
      const Row<M> xi = ldg_row<M>(a.X, own);
      float acc[M];
#pragma unroll
      for (int q = 0; q < M; ++q) acc[q] = 0.0f;
      float lf = 0.0f;
      if (FAST) {
        if (hdr.y == 0) ell_columns<M, FA, FR, true, 0, false>(a, Xt, cols + k * row_bytes, lane, W, cnt, xi, acc, lf);
        else ell_columns<M, FA, FR, true, 1, false>(a, Xt, cols + k * row_bytes, lane, W, cnt, xi, acc, lf);
        const float cc = hdr.y == 0 ? c_att : a.inv_p;  // the class constant of f'/(p d), once per lane-slot
#pragma unroll
        for (int q = 0; q < M; ++q) acc[q] *= cc;
      } else if (__all_sync(kFull, cnt == W)) {  // warp-uniform: no pads in this row
        ell_columns<M, FA, FR, false, 2, false>(a, Xt, cols + k * row_bytes, lane, W, cnt, xi, acc, lf);
      } else {
        ell_columns<M, FA, FR, false, 2, true>(a, Xt, cols + k * row_bytes, lane, W, cnt, xi, acc, lf);
      }
      if (!(ow >> 31)) red_row<M>(a.grad, own, acc);
      lrec += lf;
    }
    lsum += (double)lrec;
    // every lane's loads of this slot have returned (their consumers above have issued): refill it
    __syncwarp();
    if (lane == 0 && t2 < wt1) issue(o0, o1, s);
  }
  if (first && wt0 < wt1) { enter_bucket(); first = false; }
  while (seg_end < wt1) { ++bkt; enter_bucket(); }
  {
    double v1[1] = {lsum};
    block_sum<1>(v1, red);
    // every undirected edge was seen from both ends
    if (threadIdx.x == 0) a.loss_partials[blockIdx.x] = v1[0] * (FAST ? 0.5 * 0.6931471805599453 : 0.5);
  }
}

size_t ell_smem_bytes(int rb, int m) {
  return (size_t)((size_t)1 << rb) * m * sizeof(float) + (size_t)2 * kEllWarps * kEllSlotBytes +
         (size_t)(2 * kEllWarps + 2) * sizeof(uint64_t) + 32 * sizeof(double);
}

// compile-time function pairs of the ELL kernel
using EllPairs = FnList<Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG>, Fn1<MDE_FN_P_QUADRATIC>, Fn1<MDE_FN_L_QUADRATIC>,
                        Fn1<MDE_FN_L_HUBER>>;

const void* select_kernel(const mde_edges* e, int m) {
  const bool fast = fast_log1p_log(e->fn, e->precise);
  return with_small_m(m, [&](auto mc) {
    constexpr int M = decltype(mc)::value;
    return select_fn<M, 0>(e->fn, fast, EllPairs{}, [](auto f) {
      using F = decltype(f);
      return reinterpret_cast<const void*>(&distortion_ell_kernel<M, F::FA, F::FR, F::FAST>);
    });
  });
}

}  // namespace

namespace mde {

void ell_free(mde_edges* e) {
  cudaFree(e->ell_rec); cudaFree(e->ell_off); cudaFree(e->ell_bkt_tile); cudaFree(e->ell_bkt_wt0);
  cudaFree(e->ell_cta_desc);
  e->ell_rec = nullptr; e->ell_off = nullptr; e->ell_bkt_tile = nullptr; e->ell_bkt_wt0 = nullptr;
  e->ell_cta_desc = nullptr;
}

bool ell_supported(int64_t n, int m) {
  if (m < 1 || m > 4 || n >= (1ll << 24)) return false;
  const int rb = tile_rb(m);
  const int64_t R = 1ll << rb;
  return ((n + R - 1) >> rb) <= 32 && (R - 1) * 4 * m <= 65535 && ell_smem_bytes(rb, m) <= kMaxDynSmem;
}

// ------------------------------------------------------------------------------------------
// device builder: the same layout as ell_build_host, bit for bit, from device-resident src / dst / par0
//   1. key = (neighbour tile, class, owner) of the 2p directed entries + a histogram of the groups
//   2. stable radix sort of the entry ids by key (edge order survives inside a group, like the host's counting sort)
//   3. scan of the group counts, lane-slots of <= 8 entries per group, histogram of their lengths per (tile, class)
//   4. stable radix sort of the lane-slots by (tile, class, longest first)
//   5. the 9-bin histograms go to the host, ell_plan lays the records out, one block per record fills it
// ------------------------------------------------------------------------------------------
struct EllDev {
  unsigned char* rec = nullptr;
  EllPlan plan;
  int rb = 0;
  int64_t nentries = 0;
};

}  // namespace mde
namespace {

__global__ void ell_keys_kernel(const int32_t* __restrict__ src, const int32_t* __restrict__ dst,
                                const float* __restrict__ par0, int push_pull, int64_t p2, int64_t n, int rb,
                                uint32_t* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t* __restrict__ gcount) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p2) return;
  const int64_t e = k >> 1;
  const int s = src[e], d = dst[e];
  const int own = (k & 1) ? d : s, nbr = (k & 1) ? s : d;
  const uint32_t cls = (push_pull && !(par0[e] >= 0.0f)) ? 1u : 0u;
  const uint32_t key = (uint32_t)((((int64_t)(nbr >> rb) * 2 + cls) * n) + own);
  keys[k] = key;
  vals[k] = (uint32_t)k;
  atomicAdd(gcount + key, 1u);
}

__global__ void ell_group_slots_kernel(const uint32_t* __restrict__ gcount, int64_t ng, uint32_t* __restrict__ gslots) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g < ng) gslots[g] = (gcount[g] + (uint32_t)kEllWmax - 1u) / (uint32_t)kEllWmax;
}

// one thread per group: its lane-slots (first entry, owner, length), their sort key and the length histogram
__global__ void ell_slots_kernel(const uint32_t* __restrict__ gcount, const uint32_t* __restrict__ gstart,
                                 const uint32_t* __restrict__ gslot0, int64_t ng, int64_t n,
                                 uint32_t* __restrict__ slot_first, uint32_t* __restrict__ slot_ownlen,
                                 uint32_t* __restrict__ skey, uint32_t* __restrict__ sval, uint32_t* __restrict__ shist) {
  const int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= ng) return;
  const uint32_t c = gcount[g];
  if (c == 0) return;
  const uint32_t tc = (uint32_t)(g / n), own = (uint32_t)(g % n);
  uint32_t a = gstart[g], j = gslot0[g];
  for (uint32_t left = c; left > 0; ++j) {
    const uint32_t len = left < (uint32_t)kEllWmax ? left : (uint32_t)kEllWmax;
    slot_first[j] = a;
    slot_ownlen[j] = own | (len << 24);
    skey[j] = tc * 8u + ((uint32_t)kEllWmax - len);
    sval[j] = j;
    atomicAdd(shist + tc * 9u + len, 1u);
    a += len;
    left -= len;
  }
}

// one block per record, one thread per lane-slot position
__global__ void ell_fill_kernel(const uint32_t* __restrict__ rec_off, const int32_t* __restrict__ rec_hdr,
                                const int32_t* __restrict__ rec_slot0, const uint32_t* __restrict__ sorted_slot,
                                const uint32_t* __restrict__ slot_first, const uint32_t* __restrict__ slot_ownlen,
                                const uint32_t* __restrict__ sorted_entry, const int32_t* __restrict__ src,
                                const int32_t* __restrict__ dst, const float* __restrict__ par0, int rb, int row_bytes,
                                unsigned char* __restrict__ rec) {
  const int64_t t = blockIdx.x;
  const int W = rec_hdr[4 * t], K = rec_hdr[4 * t + 2], ns = rec_hdr[4 * t + 3];
  unsigned char* r = rec + ((size_t)rec_off[t] << 4);
  const int i = threadIdx.x;
  if (i < 4) reinterpret_cast<int32_t*>(r)[i] = rec_hdr[4 * t + i];
  if (i >= 32 * K) return;
  const int k = i >> 5, l = i & 31;
  const bool dup = i >= ns;
  const uint32_t sidx = sorted_slot[(int64_t)rec_slot0[t] + (dup ? 0 : i)];
  const uint32_t first = slot_first[sidx], ol = slot_ownlen[sidx];
  const int len = (int)(ol >> 24);
  reinterpret_cast<uint32_t*>(r + 16)[i] = (ol & kOwnMask) | (dup ? 0x80000000u : ((uint32_t)len << 24));
  unsigned char* cb = r + 16 + 128 * K + (size_t)k * (W / 2) * kEllPair;
  const uint32_t rmask = (1u << rb) - 1u;
  for (int e = 0; e < W; ++e) {
    const bool real = !dup && e < len;
    const uint32_t id = sorted_entry[first + (uint32_t)(e < len ? e : len - 1)];
    const uint32_t edge = id >> 1;
    const int nbr = (id & 1u) ? src[edge] : dst[edge];
    reinterpret_cast<float*>(cb + (e / 2) * kEllPair)[2 * l + (e & 1)] = real ? par0[edge] : 0.0f;
    reinterpret_cast<uint16_t*>(cb + (e / 2) * kEllPair + 256)[2 * l + (e & 1)] =
        (uint16_t)(((uint32_t)nbr & rmask) * (uint32_t)row_bytes);
  }
}

}  // namespace
namespace mde {

int ell_build_device(int64_t n, int64_t p, int m, const int32_t* src, const int32_t* dst, const float* par0,
                     int push_pull, int rb, int max_cta, EllDev& out, cudaStream_t st) {
  int rc = ell_check_shape(n, p, m, rb);
  if (rc) return rc;
  const int64_t R = 1ll << rb, ndt = (n + R - 1) >> rb, ng = ndt * 2 * n, p2 = 2 * p;
  const int nh = (int)(ndt * 2 * 9);
  uint32_t *keys_in = nullptr, *keys_out = nullptr, *vals_in = nullptr, *vals_out = nullptr;
  uint32_t *gcount = nullptr, *gstart = nullptr, *gslots = nullptr, *gslot0 = nullptr;
  uint32_t *slot_first = nullptr, *slot_ownlen = nullptr, *skey = nullptr, *sval = nullptr, *skey_o = nullptr,
           *sval_o = nullptr, *shist = nullptr, *d_off = nullptr;
  int32_t *d_hdr = nullptr, *d_slot0 = nullptr;
  void* tmp = nullptr;
  size_t tmp_bytes = 0, need = 0;
  std::vector<uint32_t> hist((size_t)nh, 0u);
  uint32_t tail[2] = {0, 0};
  int64_t nslots = 0;
  const int tb = 256;
#define TRY(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { rc = (int)_e; goto done; } } while (0)
  TRY(cudaMalloc(&keys_in, 4 * p2)); TRY(cudaMalloc(&keys_out, 4 * p2));
  TRY(cudaMalloc(&vals_in, 4 * p2)); TRY(cudaMalloc(&vals_out, 4 * p2));
  TRY(cudaMalloc(&gcount, 4 * ng)); TRY(cudaMalloc(&gstart, 4 * ng));
  TRY(cudaMalloc(&gslots, 4 * ng)); TRY(cudaMalloc(&gslot0, 4 * ng));
  TRY(cudaMalloc(&shist, 4 * nh));
  TRY(cudaMemsetAsync(gcount, 0, 4 * ng, st));
  TRY(cudaMemsetAsync(shist, 0, 4 * nh, st));
  ell_keys_kernel<<<ceil_div_i64(p2, tb), tb, 0, st>>>(src, dst, par0, push_pull, p2, n, rb, keys_in, vals_in, gcount);
  ++g_launch_count;
  TRY(cudaPeekAtLastError());
  // workspace: the largest of the four CUB calls
  TRY(cub::DeviceRadixSort::SortPairs(nullptr, need, keys_in, keys_out, vals_in, vals_out, (int)p2, 0, bits_for((uint64_t)ng), st));
  tmp_bytes = need;
  TRY(cub::DeviceScan::ExclusiveSum(nullptr, need, gcount, gstart, (int)ng, st));
  tmp_bytes = std::max(tmp_bytes, need);
  TRY(cudaMalloc(&tmp, tmp_bytes));
  need = tmp_bytes;
  TRY(cub::DeviceRadixSort::SortPairs(tmp, need, keys_in, keys_out, vals_in, vals_out, (int)p2, 0, bits_for((uint64_t)ng), st));
  need = tmp_bytes;
  TRY(cub::DeviceScan::ExclusiveSum(tmp, need, gcount, gstart, (int)ng, st));
  ell_group_slots_kernel<<<ceil_div_i64(ng, tb), tb, 0, st>>>(gcount, ng, gslots);
  ++g_launch_count;
  TRY(cudaPeekAtLastError());
  need = tmp_bytes;
  TRY(cub::DeviceScan::ExclusiveSum(tmp, need, gslots, gslot0, (int)ng, st));
  TRY(cudaMemcpyAsync(&tail[0], gslot0 + (ng - 1), 4, cudaMemcpyDeviceToHost, st));
  TRY(cudaMemcpyAsync(&tail[1], gslots + (ng - 1), 4, cudaMemcpyDeviceToHost, st));
  TRY(cudaStreamSynchronize(st));
  nslots = (int64_t)tail[0] + (int64_t)tail[1];
  if (nslots < 1 || nslots >= (1ll << 31)) { rc = MDE_E_UNSUPPORTED; goto done; }
  TRY(cudaMalloc(&slot_first, 4 * nslots)); TRY(cudaMalloc(&slot_ownlen, 4 * nslots));
  TRY(cudaMalloc(&skey, 4 * nslots)); TRY(cudaMalloc(&sval, 4 * nslots));
  TRY(cudaMalloc(&skey_o, 4 * nslots)); TRY(cudaMalloc(&sval_o, 4 * nslots));
  ell_slots_kernel<<<ceil_div_i64(ng, tb), tb, 0, st>>>(gcount, gstart, gslot0, ng, n, slot_first, slot_ownlen, skey, sval, shist);
  ++g_launch_count;
  TRY(cudaPeekAtLastError());
  {
    size_t need2 = 0;
    const int sbits = bits_for((uint64_t)(ndt * 2 * 8));
    TRY(cub::DeviceRadixSort::SortPairs(nullptr, need2, skey, skey_o, sval, sval_o, (int)nslots, 0, sbits, st));
    if (need2 > tmp_bytes) { cudaFree(tmp); tmp = nullptr; TRY(cudaMalloc(&tmp, need2)); tmp_bytes = need2; }
    need2 = tmp_bytes;
    TRY(cub::DeviceRadixSort::SortPairs(tmp, need2, skey, skey_o, sval, sval_o, (int)nslots, 0, sbits, st));
  }
  TRY(cudaMemcpyAsync(hist.data(), shist, 4 * nh, cudaMemcpyDeviceToHost, st));
  TRY(cudaStreamSynchronize(st));
  rc = ell_plan(hist.data(), ndt, max_cta, out.plan);
  if (rc) goto done;
  if (out.plan.nslots != nslots) { rc = MDE_E_INVALID; goto done; }
  {
    const EllPlan& pl = out.plan;
    TRY(cudaMalloc(&out.rec, (size_t)pl.rec_bytes));
    TRY(cudaMalloc(&d_off, 4 * (pl.nrec + 1)));
    TRY(cudaMalloc(&d_hdr, 16 * pl.nrec));
    TRY(cudaMalloc(&d_slot0, 4 * pl.nrec));
    TRY(cudaMemcpyAsync(d_off, pl.rec_off.data(), 4 * (pl.nrec + 1), cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(d_hdr, pl.rec_hdr.data(), 16 * pl.nrec, cudaMemcpyHostToDevice, st));
    TRY(cudaMemcpyAsync(d_slot0, pl.rec_slot0.data(), 4 * pl.nrec, cudaMemcpyHostToDevice, st));
    TRY(cudaMemsetAsync(out.rec, 0, (size_t)pl.rec_bytes, st));
    ell_fill_kernel<<<(unsigned)pl.nrec, 128, 0, st>>>(d_off, d_hdr, d_slot0, sval_o, slot_first, slot_ownlen, vals_out, src,
                                                       dst, par0, rb, 4 * m, out.rec);
    ++g_launch_count;
    TRY(cudaPeekAtLastError());
    TRY(cudaStreamSynchronize(st));
    out.rb = rb; out.nentries = p2;
  }
done:
  cudaFree(keys_in); cudaFree(keys_out); cudaFree(vals_in); cudaFree(vals_out); cudaFree(gcount); cudaFree(gstart);
  cudaFree(gslots); cudaFree(gslot0); cudaFree(slot_first); cudaFree(slot_ownlen); cudaFree(skey); cudaFree(sval);
  cudaFree(skey_o); cudaFree(sval_o); cudaFree(shist); cudaFree(d_off); cudaFree(d_hdr); cudaFree(d_slot0); cudaFree(tmp);
  if (rc != 0) { cudaFree(out.rec); out.rec = nullptr; }
  return rc;
#undef TRY
}

// Called on a finished sorted-SoA layout (kind 0): builds the ELL records from its src / dst / par0 on the device
// (MDE_B200_ELL_BUILD=host: copies them to the host and runs ell_build_host, the builder the CPU tests cover; both give the
// same bytes); on success the layout becomes kind 3.  Returns 0, MDE_E_UNSUPPORTED (layout stays kind 0) or an error.
int ell_build(mde_edges* e, const mde_fn_t* fn, int m, cudaStream_t st) {
  if (e->kind != kSoa || e->has_par1 || e->det || m < 1 || m > 4) return MDE_E_UNSUPPORTED;
  const int rb = tile_rb(m);
  if (ell_smem_bytes(rb, m) > kMaxDynSmem) return MDE_E_UNSUPPORTED;
  const int64_t p = e->p, n = e->n;
  int rc = ell_check_shape(n, p, m, rb);
  if (rc) return rc;
  if ((rc = allow_max_smem(select_kernel(e, m)))) return rc;
  const char* bev = getenv("MDE_B200_ELL_BUILD");
  const bool on_host = bev && !strcmp(bev, "host");
  EllHost h;
  EllDev d;
  const EllPlan* pl = nullptr;
  if (on_host) {
    std::vector<int32_t> hs((size_t)p), hd((size_t)p);
    std::vector<float> hw((size_t)p);
    MDE_CUDA_TRY(cudaMemcpyAsync(hs.data(), e->src, sizeof(int32_t) * p, cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaMemcpyAsync(hd.data(), e->dst, sizeof(int32_t) * p, cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaMemcpyAsync(hw.data(), e->par0, sizeof(float) * p, cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaStreamSynchronize(st));
    rc = ell_build_host(n, p, m, hs.data(), hd.data(), hw.data(), fn->push_pull, rb, kNumSMs, h);
    if (rc) return rc;
    pl = &h.plan;
    cudaError_t ce = cudaMalloc(&e->ell_rec, h.rec.size());
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(e->ell_rec, h.rec.data(), h.rec.size(), cudaMemcpyHostToDevice, st);
    if (ce != cudaSuccess) { ell_free(e); return (int)ce; }
  } else {
    rc = ell_build_device(n, p, m, e->src, e->dst, e->par0, fn->push_pull, rb, kNumSMs, d, st);
    if (rc) return rc;
    pl = &d.plan;
    e->ell_rec = d.rec;
  }
  const int nbkt = (int)pl->bkt_tile.size();
#define UP(dst, vec, T)                                                                              \
  do {                                                                                               \
    cudaError_t _e = cudaMalloc(&(dst), sizeof(T) * (vec).size());                                   \
    if (_e == cudaSuccess) _e = cudaMemcpyAsync((dst), (vec).data(), sizeof(T) * (vec).size(), cudaMemcpyHostToDevice, st); \
    if (_e != cudaSuccess) { ell_free(e); return (int)_e; }                                          \
  } while (0)
  UP(e->ell_off, pl->rec_off, uint32_t);
  UP(e->ell_bkt_tile, pl->bkt_tile, int32_t);
  UP(e->ell_bkt_wt0, pl->bkt_wt0, int32_t);
  std::vector<int32_t> desc((size_t)4 * pl->ncta);
  for (int c = 0; c < pl->ncta; ++c) {
    desc[4 * c] = pl->cta_wt0[c]; desc[4 * c + 1] = pl->cta_wt0[c + 1]; desc[4 * c + 2] = pl->cta_bkt0[c];
    desc[4 * c + 3] = pl->bkt_tile[(size_t)pl->cta_bkt0[c]];
  }
  UP(e->ell_cta_desc, desc, int32_t);
#undef UP
  cudaError_t se = cudaStreamSynchronize(st);  // the host vectors die with this frame
  if (se != cudaSuccess) { ell_free(e); return (int)se; }
  e->kind = kSoaEll; e->m_hint = m; e->rb = rb; e->ell_nrec = pl->nrec; e->ell_ncta = pl->ncta; e->nbkt = nbkt;
  e->nbytes += pl->rec_bytes + 4 * (pl->nrec + 1) + 4ll * (2 * nbkt + 4 * pl->ncta + 2);
  return 0;
}

int ell_launch(const mde_edges* e, const float* X, int m, float* grad, int* nblocks_out, const int* flag,
               cudaStream_t st) {
  if (e->kind != kSoaEll || m != e->m_hint || !grad) return MDE_E_UNSUPPORTED;
  const size_t smem = ell_smem_bytes(e->rb, m);
  EllArgs a;
  a.rec = e->ell_rec; a.rec_off = e->ell_off; a.bkt_tile = e->ell_bkt_tile; a.bkt_wt0 = e->ell_bkt_wt0;
  a.cta_desc = reinterpret_cast<const int4*>(e->ell_cta_desc); a.X = X; a.grad = grad;
  a.loss_partials = e->loss_partials; a.flag = flag; a.fn = e->fn; a.inv_p = 1.0f / (float)e->p_total;
  a.n = e->n; a.rb = e->rb;
  a.x_vec_ok = ((reinterpret_cast<uintptr_t>(X) & 15u) == 0) ? 1 : 0;
  return launch_persistent(select_kernel(e, m), &a, e->ell_ncta, kEllThreads, smem, nblocks_out, st);
}

}  // namespace mde

// ------------------------------------------------------------------------------------------
// host-only export for the CPU tests: build the ELL records from host arrays, no device involved
// ------------------------------------------------------------------------------------------
extern "C" {

static int ell_export(const EllPlan& pl, const unsigned char* rec_host, int rb, int64_t nentries, mde_ell_host_t* out) {
  memset(out, 0, sizeof(*out));
  auto dup = [](const void* p_, size_t bytes) -> void* {
    void* q = malloc(bytes ? bytes : 1);
    if (q && bytes) memcpy(q, p_, bytes);
    return q;
  };
  out->rec_bytes = pl.rec_bytes;
  out->nrec = pl.nrec; out->nbkt = (int32_t)pl.bkt_tile.size(); out->ncta = pl.ncta; out->tile_rows_log2 = rb;
  out->nslots = pl.nslots; out->nentries = nentries; out->npadded = pl.npadded;
  out->rec = (unsigned char*)dup(rec_host, (size_t)pl.rec_bytes);
  out->rec_off = (uint32_t*)dup(pl.rec_off.data(), 4 * pl.rec_off.size());
  out->bkt_tile = (int32_t*)dup(pl.bkt_tile.data(), 4 * pl.bkt_tile.size());
  out->bkt_wt0 = (int32_t*)dup(pl.bkt_wt0.data(), 4 * pl.bkt_wt0.size());
  out->cta_wt0 = (int32_t*)dup(pl.cta_wt0.data(), 4 * pl.cta_wt0.size());
  out->cta_bkt0 = (int32_t*)dup(pl.cta_bkt0.data(), 4 * pl.cta_bkt0.size());
  if (!out->rec || !out->rec_off || !out->bkt_tile || !out->bkt_wt0 || !out->cta_wt0 || !out->cta_bkt0) {
    mde_ell_host_free(out);
    return MDE_E_ALLOC;
  }
  return 0;
}

int mde_ell_host_layout(int64_t n_items, int64_t p, int embedding_dim, const int32_t* src, const int32_t* dst,
                        const float* par0, int push_pull, int tile_rows_log2, int max_cta, mde_ell_host_t* out) {
  if (!src || !dst || !par0 || !out) return MDE_E_INVALID;
  EllHost h;
  const int rb = tile_rows_log2 > 0 ? tile_rows_log2 : default_tile_rb(embedding_dim);
  const int rc = ell_build_host(n_items, p, embedding_dim, src, dst, par0, push_pull, rb, max_cta > 0 ? max_cta : kNumSMs, h);
  if (rc) return rc;
  return ell_export(h.plan, h.rec.data(), h.rb, h.nentries, out);
}

int mde_ell_device_layout(int64_t n_items, int64_t p, int embedding_dim, const int32_t* src, const int32_t* dst,
                          const float* par0, int push_pull, int tile_rows_log2, int max_cta, mde_ell_host_t* out,
                          void* stream) {
  if (!src || !dst || !par0 || !out) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  mde::EllDev d;
  const int rb = tile_rows_log2 > 0 ? tile_rows_log2 : default_tile_rb(embedding_dim);
  int rc = mde::ell_build_device(n_items, p, embedding_dim, src, dst, par0, push_pull, rb, max_cta > 0 ? max_cta : kNumSMs, d, st);
  if (rc) return rc;
  std::vector<unsigned char> host((size_t)d.plan.rec_bytes);
  cudaError_t ce = cudaMemcpyAsync(host.data(), d.rec, host.size(), cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  cudaFree(d.rec);
  if (ce != cudaSuccess) return (int)ce;
  return ell_export(d.plan, host.data(), d.rb, d.nentries, out);
}

void mde_ell_host_free(mde_ell_host_t* h) {
  if (!h) return;
  free(h->rec); free(h->rec_off); free(h->bkt_tile); free(h->bkt_wt0); free(h->cta_wt0); free(h->cta_bkt0);
  memset(h, 0, sizeof(*h));
}

}  // extern "C"
