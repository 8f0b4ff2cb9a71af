// mde_edges.cuh -- the device-resident edge layout and what its four kernel families share: the m <= 4 row helpers,
// the choice of compile-time function ids, the host helpers of the tile, pull and ELL builders and launches, and the
// evaluation entries by layout kind (mde_edges.cu), which the C ABI and the device solver call.
//
// Layouts (one per shard, chosen at mde_edges_create_ex):
//
//  kind 0  "sorted SoA"     src[p], dst[p], par0[p] (, par1[p]) sorted by (class, src, dst); perm[p].
//                           Any m; the m >= 5 kernels, WeightedQuadratic (par1) and very sparse graphs use it.
//
//  kind 1  "tile records"   m <= 4.  Vertices are cut into dst tiles of R rows (R * m * 8 bytes of X + gradient
//                           fit in one SM's shared memory) and src super-tiles of 2^ss rows (X + gradient of a
//                           super-tile fit in L2).  Edges are grouped into buckets (src super-tile, dst tile),
//                           inside a bucket sorted by (class, src, dst), every bucket padded to whole
//                           "warp-tiles" of 128 edges.  One warp-tile is ONE contiguous 1536-byte record
//                               int32 src[128] | int32 dst[128] | fp32 par0[128]        (pad: dst = -1)
//                           so a warp fetches it with a single cp.async.bulk (TMA) into its shared-memory slot.
//                           perm[nwt * 128] holds the caller position of every slot (-1 for pads).
//
//  kind 3  "SoA + ELL"      m <= 4, n < 2^24, <= 32 neighbour tiles: the kind-0 arrays plus the ELL pull records of
//                           mde_ell.cu (one lane per owner, 12 bytes per edge).
//
//  kind 2  "pull records"   m <= 4.  Same buckets, but every edge is stored as two DIRECTED entries (owner,
//                           neighbour) and a bucket is (owner super-tile, neighbour tile, class); records are
//                           1040 bytes: fp32 w[128] | u16 owner offset[128] | u16 neighbour offset[128] | header
//                           (mde_pull.cu).  No shared-memory atomics, one global red per owner run.
#pragma once
#include <cstdlib>
#include <type_traits>
#include <vector>

#include "mde_common.cuh"

namespace mde {
enum LayoutKind : int { kSoa = 0, kTiles = 1, kPull = 2, kSoaEll = 3 };  // mde_edges::kind (mde_edges_kind)
}

struct mde_edges {
  int64_t p = 0, n = 0, p_total = 0;
  mde::LayoutKind kind = mde::kSoa;
  // ---- kind 0 ----
  int32_t *src = nullptr, *dst = nullptr;
  float *par0 = nullptr, *par1 = nullptr;
  // ---- both ----
  int32_t* perm = nullptr;
  double* loss_partials = nullptr;  // [kMaxLossBlocks]
  mde::FnDev fn;
  int has_par1 = 0;
  int64_t nbytes = 0;
  // MDE_B200_KERNEL=precise: IEEE math in place of the MUFU forms, resolved once when the layout is created (layouts
  // built with and without it coexist)
  bool precise = false;
  int det = 0;               // deterministic mode: m <= 4 fixed point (fx), 5 <= m <= 512 the wide owner kernel
  long long* fx = nullptr;   // [n * m_hint] fixed-point accumulator (det, m_hint <= 4 only)
  unsigned* fx_max = nullptr;     // [n] det, m_hint <= 4: bits of the row's largest finite |contribution| (per evaluation)
  uint8_t* fx_lgdeg = nullptr;    // [n] det, m_hint <= 4: ceil(log2(degree)) of every row
  // sorted-SoA layout, m_hint <= 4 (and deterministic layouts with 5 <= m_hint <= 512): every edge is stored again as
  // two directed entries grouped by owner node, and the owner kernels visit each node's entries in this fixed order,
  // keep the sum in registers and write the row once (no atomics) -- a gradient that is the same bits from run to run
  uint32_t* inc = nullptr;      // [2 p] (k << 1) | (node is dst), grouped by node: src entries by k, then dst entries by k
  uint2* ent = nullptr;         // [2 p] in the order of inc: (neighbour row | (node is dst) << 31, bits of par0[k])
  int64_t* inc_off = nullptr;   // [n + 1] first entry of node i in inc / ent
  // deterministic layouts with m_hint >= 5: lists longer than kWideSeg entries are evaluated in segments (mde_edges.cu)
  int nwseg = 0, nwhub = 0;
  int4* wseg = nullptr;         // [nwseg] (node, first entry, end entry) of every segment, in node and list order
  int4* whub = nullptr;         // [nwhub] (node, first segment, end segment) of every node that has segments
  float* wpart = nullptr;       // [nwseg * m_hint] the segments' partial gradient rows
  // ---- kind 1 ----
  int m_hint = 0;          // embedding dimension the tile size was chosen for
  int rb = 0;              // log2(R): dst tile rows
  int ss = 0;              // log2(super-tile rows)
  int64_t nwt = 0;         // warp-tiles (128 slots each), padding included
  int32_t* rec = nullptr;  // nwt * 384 words
  int nbkt = 0;            // non-empty buckets
  int32_t* bkt_tile = nullptr;  // [nbkt]     dst tile of bucket b
  int32_t* bkt_wt0 = nullptr;   // [nbkt + 1] first warp-tile of bucket b
  int ncta = 0;                 // persistent grid of the tile kernel
  int32_t* cta_wt0 = nullptr;   // [ncta + 1] warp-tile range of CTA c
  int32_t* cta_bkt0 = nullptr;  // [ncta]     bucket holding cta_wt0[c]
  // ---- kind 2 (pull records, mde_pull.cu): same bucket / CTA tables, 1040-byte records of DIRECTED entries ----
  int32_t* wt_tile = nullptr;   // [nwt] neighbour tile of every warp-tile (per-edge outputs)
  int epl = 4;                  // entries per lane per warp-tile (a warp-tile holds 32 * epl entries)
  // ---- kind 3 (sorted SoA + ELL pull records, mde_ell.cu): the kind-0 arrays above stay valid ----
  unsigned char* ell_rec = nullptr;   // variable-size records (144 + 192 W bytes)
  uint32_t* ell_off = nullptr;        // [ell_nrec + 1] record offsets, units of 16 bytes
  int32_t *ell_bkt_tile = nullptr, *ell_bkt_wt0 = nullptr;
  int32_t* ell_cta_desc = nullptr;    // [ell_ncta] int4: first record, end record, first bucket, its neighbour tile
  int64_t ell_nrec = 0;
  int ell_ncta = 0;
};

namespace mde {

constexpr int kMaxLossBlocks = kNumSMs * 16;
constexpr int kWtEdges = 128;                 // slots per warp-tile
constexpr int kWtWords = 3 * kWtEdges;        // 32-bit words per record
constexpr int kWtBytes = kWtWords * 4;        // 1536
constexpr size_t kMaxDynSmem = 227u * 1024u;  // dynamic shared memory a CTA may opt in to on the H100

// ------------------------------------------------------------------------------------------
// m <= 4 rows in registers.  Rows are indexed by int, widened to int64_t, except in the ELL kernel, whose uint32_t
// rows widen to size_t.
// ------------------------------------------------------------------------------------------
template <int M> struct Row { float v[M]; };

__device__ __forceinline__ int64_t wide(int r) { return r; }
__device__ __forceinline__ size_t wide(uint32_t r) { return r; }

// row r of X (global memory, read-only path)
template <int M, typename I>
__device__ __forceinline__ Row<M> ldg_row(const float* __restrict__ X, I r) {
  Row<M> o;
  if constexpr (M == 1) { o.v[0] = __ldg(X + r); }
  else if constexpr (M == 2) { const float2 t = __ldg(reinterpret_cast<const float2*>(X) + r); o.v[0] = t.x; o.v[1] = t.y; }
  else if constexpr (M == 4) { const float4 t = __ldg(reinterpret_cast<const float4*>(X) + r); o.v[0] = t.x; o.v[1] = t.y; o.v[2] = t.z; o.v[3] = t.w; }
  else {
#pragma unroll
    for (int c = 0; c < M; ++c) o.v[c] = __ldg(X + wide(r) * M + c);
  }
  return o;
}

// A record of a stream that a kernel reads once per launch while it gathers rows of X again and again (the owner
// kernel's `ent`, `inc`, `inc_off`): ld.global.nc.L1::evict_first, so the stream is the first to leave L1.  No L2
// hint: the records stay L2-resident from one evaluation to the next.
__device__ __forceinline__ uint2 ldg_stream(const uint2* __restrict__ p) {
  uint2 o;
  asm("ld.global.nc.L1::evict_first.v2.u32 {%0, %1}, [%2];" : "=r"(o.x), "=r"(o.y) : "l"(p));
  return o;
}
__device__ __forceinline__ uint32_t ldg_stream(const uint32_t* __restrict__ p) {
  uint32_t o;
  asm("ld.global.nc.L1::evict_first.u32 %0, [%1];" : "=r"(o) : "l"(p));
  return o;
}
__device__ __forceinline__ int64_t ldg_stream(const int64_t* __restrict__ p) {
  int64_t o;
  asm("ld.global.nc.L1::evict_first.s64 %0, [%1];" : "=l"(o) : "l"(p));
  return o;
}

// row r of a shared-memory tile
template <int M>
__device__ __forceinline__ Row<M> lds_row(const float* __restrict__ Xt, int r) {
  Row<M> o;
  if constexpr (M == 2) { const float2 t = reinterpret_cast<const float2*>(Xt)[r]; o.v[0] = t.x; o.v[1] = t.y; }
  else if constexpr (M == 4) { const float4 t = reinterpret_cast<const float4*>(Xt)[r]; o.v[0] = t.x; o.v[1] = t.y; o.v[2] = t.z; o.v[3] = t.w; }
  else {
#pragma unroll
    for (int c = 0; c < M; ++c) o.v[c] = Xt[r * M + c];
  }
  return o;
}

// the row at BYTE offset `off` of a shared-memory tile (the ELL records store byte offsets).  It fills the caller's
// array: returned as a Row, the m = 3 ELL kernel of the run-time table compiles to different code.
template <int M>
__device__ __forceinline__ void lds_row_at(const float* __restrict__ Xt, uint32_t off, float (&o)[M]) {
  const unsigned char* q = reinterpret_cast<const unsigned char*>(Xt) + off;
  if constexpr (M == 2) { const float2 t = *reinterpret_cast<const float2*>(q); o[0] = t.x; o[1] = t.y; }
  else if constexpr (M == 4) { const float4 t = *reinterpret_cast<const float4*>(q); o[0] = t.x; o[1] = t.y; o[2] = t.z; o[3] = t.w; }
  else {
#pragma unroll
    for (int c = 0; c < M; ++c) o[c] = reinterpret_cast<const float*>(q)[c];
  }
}

// G[r] += sgn * v as one vector red (SASS REDG.E.ADD.F32x2 / x4) where the row width allows it
template <int M, typename I>
__device__ __forceinline__ void red_row(float* __restrict__ G, I r, const float (&v)[M], float sgn = 1.0f) {
  if constexpr (M == 1) red_add(G + r, sgn * v[0]);
  else if constexpr (M == 2) red_add_v2(G + 2 * wide(r), sgn * v[0], sgn * v[1]);
  else if constexpr (M == 4) red_add_v4(G + 4 * wide(r), sgn * v[0], sgn * v[1], sgn * v[2], sgn * v[3]);
  else {
#pragma unroll
    for (int c = 0; c < M; ++c) red_add(G + wide(r) * M + c, sgn * v[c]);
  }
}

// ------------------------------------------------------------------------------------------
// which kernel runs (host).  Every family instantiates its kernels for a few (attractive, repulsive) function pairs
// with compile-time ids, and for the run-time table.
// ------------------------------------------------------------------------------------------
// Fn<FA, FR>: FA != FR is PushAndPull(FA, FR), FA == FR one function without PushAndPull, Fn<-1, -1> the run-time
// table.  FAST: the MUFU form of the recipe default PushAndPull(Log1p(1.5), Log(1)).
template <int FA_, int FR_, bool FAST_ = false>
struct Fn {
  static constexpr int FA = FA_, FR = FR_;
  static constexpr bool FAST = FAST_;
  static bool matches(const FnDev& fn) {
    return FA != FR ? (fn.push_pull && fn.fn_att == FA && fn.fn_rep == FR) : (!fn.push_pull && fn.fn_att == FA);
  }
};
template <int F> using Fn1 = Fn<F, F>;
template <class... P> struct FnList {};

// The recipe default runs on the MUFU form unless MDE_B200_KERNEL=precise asked for IEEE math everywhere.
inline bool fast_log1p_log(const FnDev& fn, bool precise) {
  return fn.push_pull && fn.fn_att == MDE_FN_P_LOG1P && fn.fn_rep == MDE_FN_P_LOG && fn.a0 == 1.5f && fn.r0 == 1.0f &&
         !precise;
}

// launch(P{}) for the first pair P of the list that matches fn, launch(Fn<-1, -1>{}) when none does
template <class F>
auto select_pair(const FnDev&, FnList<>, F&& launch) { return launch(Fn<-1, -1>{}); }
template <class P0, class... P, class F>
auto select_pair(const FnDev& fn, FnList<P0, P...>, F&& launch) {
  return P0::matches(fn) ? launch(P0{}) : select_pair(fn, FnList<P...>{}, launch);
}

// Returns launch(Fn<...>{}) for the kernel that evaluates fn.  Only the fused evaluation at m = 2 and 3 has
// compile-time ids: the MUFU kernel when `fast` (families without one pass false), else the pair of the family's list
// that matches fn.  Everything else runs on the run-time table.
template <int M, int MODE, class... P, class F>
auto select_fn(const FnDev& fn, bool fast, FnList<P...> pairs, F&& launch) {
  if constexpr (MODE == 0 && (M == 2 || M == 3)) {
    if (fast) return launch(Fn<MDE_FN_P_LOG1P, MDE_FN_P_LOG, true>{});
    return select_pair(fn, pairs, launch);
  }
  return launch(Fn<-1, -1>{});
}

// f(std::integral_constant<int, M>{}) for the row width m = M = 1..4 of the tile, pull and ELL kernels; nullptr for
// any other m
template <class F>
const void* with_small_m(int m, F&& f) {
  switch (m) {
    case 1: return f(std::integral_constant<int, 1>{});
    case 2: return f(std::integral_constant<int, 2>{});
    case 3: return f(std::integral_constant<int, 3>{});
    case 4: return f(std::integral_constant<int, 4>{});
  }
  return nullptr;
}

// ------------------------------------------------------------------------------------------
// host helpers of the tile, pull and ELL layouts
// ------------------------------------------------------------------------------------------
inline int env_int(const char* name, int dflt) {
  const char* e = getenv(name);
  return e ? atoi(e) : dflt;
}

inline int bits_for(uint64_t maxval) {  // bits needed to hold values 0..maxval
  int b = 1;
  while (b < 64 && (maxval >> b) != 0) ++b;
  return b;
}

// log2 of the rows of one shared-memory tile: 8192 rows for m <= 2, else 4096 (a 64 KB X tile at m = 2 and 4, 48 KB
// at m = 3; the tile-record kernel adds a gradient tile of the same size).  MDE_B200_TILE_RB=8..15 overrides it.
inline int default_tile_rb(int m) { return (m <= 2) ? 13 : 12; }
inline int tile_rb(int m) {
  const int r = env_int("MDE_B200_TILE_RB", 0);
  return (r >= 8 && r <= 15) ? r : default_tile_rb(m);
}

// Dynamic shared memory above 48 KB needs an opt-in per kernel.  Done once per kernel, when a layout is built for the
// kernels it will launch, so never for the first time inside a stream capture.  No kernel (nullptr): MDE_E_UNSUPPORTED.
int allow_max_smem(const void* kernel);

// The tile and pull builders' persistent grid: up to one CTA per SM, CTA c walks warp-tiles [cta_wt0[c], cta_wt0[c + 1])
// and starts in bucket cta_bkt0[c].  Returns the number of CTAs.
int split_ctas(int64_t nwt, const std::vector<int32_t>& bkt_wt0, std::vector<int32_t>& cta_wt0,
               std::vector<int32_t>& cta_bkt0);

// Launches `kernel` with its one argument struct `args` on the persistent grid (after allow_max_smem).
int launch_persistent(const void* kernel, void* args, int ncta, int threads, size_t smem, int* nblocks_out,
                      cudaStream_t st);

// ------------------------------------------------------------------------------------------
// evaluations on any layout kind (mde_edges.cu).  flag: device gate, the kernels return at once when *flag == 0
// (nullptr: always run).
// ------------------------------------------------------------------------------------------
// MODE 0: fused value + gradient; 1: value only; 2: gradient from caller-ordered per-edge coefficients `gext`.
// Modes 0 and 1 leave *nblocks_out per-block loss partials in e->loss_partials.
int evaluate(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext, int* nblocks_out,
             const int* flag, cudaStream_t st);
// distances and distortions (either may be nullptr) in the caller's edge order
int edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions, const int* flag,
                 cudaStream_t st);

// tile kernel (mde_tiled.cu)
int tiled_build(mde_edges* e, const int64_t* edges, const float* par0, const mde_fn_t* fn, int embedding_dim,
                cudaStream_t st);
void tiled_free(mde_edges* e);
int tiled_launch(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                 int* nblocks_out, const int* flag, cudaStream_t st);
int tiled_edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions,
                       const int* flag, cudaStream_t st);

// pull kernel (mde_pull.cu)
int pull_build(mde_edges* e, const int64_t* edges, const float* par0, const mde_fn_t* fn, int embedding_dim,
               cudaStream_t st);
void pull_free(mde_edges* e);
int pull_launch(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                int* nblocks_out, const int* flag, cudaStream_t st);
int pull_edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions,
                      const int* flag, cudaStream_t st);

// ELL pull kernel (mde_ell.cu): fused value + gradient only; everything else runs on the sorted-SoA kernels
bool ell_supported(int64_t n_items, int embedding_dim);  // shape accepted by the ELL builder (before any allocation)
int ell_build(mde_edges* e, const mde_fn_t* fn, int embedding_dim, cudaStream_t st);
void ell_free(mde_edges* e);
int ell_launch(const mde_edges* e, const float* X, int m, float* grad, int* nblocks_out, const int* flag,
               cudaStream_t st);

}  // namespace mde
