// mde_knn.cu -- exact k-nearest neighbours of the rows of a data matrix (SURVEY section 8 row f3).
//
// Replaces the neighbour search of pymde/preprocess/data_matrix.py:91-178 (scikit-learn brute force below 10 000
// rows, pynndescent above) by an exact search whose cross terms run on the Hopper tensor cores (wgmma):
//
//   prep     X (n x d fp32) -> Xh, Xl (n_pad x K_pad bf16, x = hi + lo to 2^-16), ||x||^2 (fp32; +inf on padding)
//   tiles    one CTA per 128 query rows sweeps ALL candidates in tiles of 128:
//              a producer warp stages 64-wide K blocks of the hi and lo parts of both operands in shared memory with
//              TMA (cp.async.bulk.tensor.2d, 128-byte swizzle; 2 stages x 64 KB, mbarrier pipeline), and two consumer
//              warpgroups (64 query rows each) issue
//              wgmma.mma_async.m64n128k16.f32.bf16.bf16  D[64 x 128] += Ah Bh^T + Ah Bl^T + Al Bh^T   (fp32 registers),
//              stage the finished accumulator in shared memory, form ||x||^2 - 2 q.x and keep, per query row, the
//              KK = 32 smallest in thread-private lists (two threads per row, merged at the end).  The n x n distance
//              matrix never exists.
//   re-rank  exact fp32 sum (q - x)^2 of the KK candidates of a row (one warp per row), k smallest, ascending.
//
// The prep works on the column-centred values x^ = fl(x - mu) (mu: fp64 column sums in a fixed order, rounded to
// fp32), which removes a global offset from the scores, unless the raw rows give the smaller error bound (knn_centre:
// a 16-bit element near the origin is its own exact operand); the re-rank reads the raw rows.  The bf16 x 3 split still
// leaves an error of ~2^-16 |q^||x^| on a cross term, which is noise when clusters lie far apart against their spread.
//   certify  a proven bound E(q) on the score error (knn_certify_kernel) shows, row by row, that no row the tiles did
//            not keep can enter the re-ranked list;
//   direct   the rows that fail are searched over all n rows with the re-rank's arithmetic (knn_direct_kernel).
// So the result is the k smallest (fp32 distance, index) pairs of a brute-force fp32 search, ties included, on every
// input; the certificate only decides how much of it the tensor cores do.  k <= 24.
//
// mde_knn_wide (24 < k <= 64): knn_wide_tile_kernel does the same sweep for 64 query rows per CTA with one consumer
// warpgroup and keeps KK = 96 candidates per row in shared memory (mde_knn_select.cuh); knn_wide_rerank_kernel
// re-ranks all 96 with the arithmetic above.  mde_knn_long (k <= 256) is the same kernel with KK = 288 and candidate
// tiles of 64 (wgmma.m64n64k16), so that its lists fit in shared memory; knn_long_rerank_kernel re-ranks all 288.
//
// mde_knn_rows / mde_knn16_rows search a range of query rows against all n rows with the narrow or wide tiles (every
// full search is the range [0, n)).  When the query tiles leave SMs idle the candidate tiles are split into S slices
// (blockIdx.y; S from mde_logic.h::knn_slices), each CTA keeps its own top-KK, knn_merge_rerank_kernel re-ranks the
// S KK candidates of a row exactly, and the certificate takes the smallest of the S worst kept scores (DESIGN 11.8).
// mde_knn_long_rows / mde_knn16_long_rows / mde_knn8_long_rows split the long search the same way; their merge
// (knn_long_select_kernel) radix-selects the full search's 288 candidates from a row's S 288 before the long re-rank.
//
// 16-bit input (mde_knn16, mde_knn16_wide, mde_knn16_long: IEEE fp16 or bf16, read without an fp32 copy).  The element
// type T is a template parameter of every kernel above.  The prep copies X into a zero-padded operand of its own type
// (no lo part) and writes the norms with the arithmetic of the fp32 prep on the upcast values; the tile kernels issue
// one wgmma per k16 step, bf16 x bf16 or fp16 x fp16, on the stage layout and barrier protocol of the fp32 route with
// the lo slots left empty; the re-rank converts each element to fp32 as it reads it.  For bf16 input the lo operand of
// the fp32 route is exactly zero, so its two extra products add exact zeros and the candidate lists are the same; an
// fp16 product is exact in fp32, so the cross terms differ from the split's by rounding alone, and the re-rank of the
// unchanged arithmetic gives the bits of the fp32 route on X.float() (near-ties at the list's edge aside, DESIGN
// section 11.7).
//
// 8-bit input (mde_knn8, mde_knn8_wide, mde_knn8_long, mde_knn8_rows: uint8 or int8, read without an fp32 copy).  The
// element is its own operand, exact wherever the data sits, so nothing is centred: the prep copies X into a zero-padded
// operand (K blocks of 128 elements, one 128-byte swizzle row) and writes exact int32 squared norms (INT_MAX on padded
// rows); the tile kernels issue one wgmma.m64n{128,64}k32.s32.{u8,s8} per 32 features, four per K block, on the same
// stage layout, and rank candidates by the exact integer score ||y||^2 - 2 <q, y>.  Every accumulator, norm and score
// is exact in int32 up to d_max (knn8_max_d); the entries refuse wider matrices.  The lists hold the KK smallest exact
// distances, the re-rank is the fp32 one, and the certificate compares the k-th re-ranked distance with the exact
// KK-th (knn_certify_kernel), so the result is again the brute-force fp32 result on X.float() (DESIGN section 11.9).
//
// Hangs are not an option on a shared GPU: every mbarrier wait is bounded (mde_tma.cuh) and traps.
#include <cuda.h>  // CUtensorMap and its enums (types only: the encoder is fetched with cudaGetDriverEntryPoint)
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <climits>
#include <cstdint>
#include <cstdlib>
#include <type_traits>

#include "mde_common.cuh"
#include "mde_knn_select.cuh"
#include "mde_logic.h"
#include "mde_tma.cuh"
#include "mde_wgmma.cuh"

using namespace mde;

namespace {

constexpr int kTileM = 128;                 // query rows per CTA (two warpgroups of 64)
constexpr int kTileN = 128;                 // candidates per tile = wgmma N
constexpr int kStages = 2;
constexpr int kKK = kNarrowKK;              // candidates kept per row before the exact re-rank (32)
constexpr int kMaxK = 24;
constexpr int kRowBytes = 128;              // one K block: a 128-byte swizzle row (64 16-bit or 128 8-bit elements)
constexpr int kKSteps = kRowBytes / 32;     // wgmma K steps per block: k16 on 16-bit operands, k32 on 8-bit ones
constexpr int kOpBytes = 128 * kRowBytes;   // 16 KB: one 128-row operand block (hi or lo)
constexpr int kStageBytes = 4 * kOpBytes;   // A hi, A lo, B hi, B lo = 64 KB
constexpr int kConsumerWarps = 8;           // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kAccStride = kTileN + 2;      // floats per staged accumulator row: the scan's column reads are conflict-free
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /* alignment slack */ + kTileM * kAccStride * 4 +
                           2 * kTileN * 4 /* norms */ + 64 /* barriers */;
static_assert(kTileM == 128 && kTileN == 128, "one TMA box (64 x 128) serves both operands");
static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

// wide (k <= 64) and long (k <= 256) searches: 64 query rows per CTA, one consumer warpgroup, running top-KK lists in
// shared memory, candidate tiles of TN = 128 (wide) or 64 (long) rows
constexpr int kWideTileM = 64;
constexpr int kAOpBytes = kWideTileM * kRowBytes;          // 8 KB: one 64-row query operand block (hi or lo)
constexpr int kWideConsumerWarps = 4;                       // warps 0-3: one consumer warpgroup; warp 4: TMA producer
constexpr int kWideThreads = (kWideConsumerWarps + 1) * 32;
constexpr int kLongTileN = 64;

template <int TN>
constexpr int kWideStageBytes = 2 * kAOpBytes + 2 * TN * kRowBytes;  // A hi, A lo, B hi, B lo
template <int KK, int TN>
constexpr int kWideSmemBytes = kStages * kWideStageBytes<TN> + 1024 /* alignment slack */ +
                               kWideTileM * (TN + 2) * 4 /* accumulators */ + TN * 4 /* norms */ +
                               kWideTileM * WideList<KK>::kStride * 8 /* lists */ + 64 /* barriers */;
// wide: 2 x 48 KB stages, 33 KB accumulators, 49 KB lists.  long: 148.5 KB of lists leave room for 2 x 32 KB stages
// of 64-wide candidate tiles and a 16.5 KB accumulator (232 256 bytes in all)
static_assert(kWideSmemBytes<kWideKK, kTileN> <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
static_assert(kWideSmemBytes<kLongKK, kLongTileN> <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

// Query ranges and candidate slices: QueryRange, kMaxSlices (mde_knn_select.cuh).  The dense searches take base = lo
// rounded down to 128, so that every query box also lies inside the padded operand.

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers (tensor TMA); mbarriers come from mde_tma.cuh, wgmma from mde_wgmma.cuh
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// The tensor-core operand of an element type: fp32 is split into bf16 hi and lo parts (three products per k16 step),
// a 16-bit or 8-bit element is its own operand (one product).  Acc: the type of the accumulators, norms and scores
// (int32 for 8-bit operands, whose products and sums are exact integers); kBlockK: elements per 128-byte K block.
template <class T>
struct Operand {
  using type = __nv_bfloat16;
  using Acc = float;
  static constexpr bool kSplit = true;
  static constexpr int kBlockK = 64;
  static constexpr CUtensorMapDataType kMapType = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
};
template <>
struct Operand<__nv_bfloat16> {
  using type = __nv_bfloat16;
  using Acc = float;
  static constexpr bool kSplit = false;
  static constexpr int kBlockK = 64;
  static constexpr CUtensorMapDataType kMapType = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
};
template <>
struct Operand<__half> {
  using type = __half;
  using Acc = float;
  static constexpr bool kSplit = false;
  static constexpr int kBlockK = 64;
  static constexpr CUtensorMapDataType kMapType = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
};
template <>
struct Operand<uint8_t> {
  using type = uint8_t;
  using Acc = int;
  static constexpr bool kSplit = false;
  static constexpr int kBlockK = 128;
  static constexpr CUtensorMapDataType kMapType = CU_TENSOR_MAP_DATA_TYPE_UINT8;
};
template <>
struct Operand<int8_t> {
  using type = int8_t;
  using Acc = int;
  static constexpr bool kSplit = false;
  static constexpr int kBlockK = 128;
  static constexpr CUtensorMapDataType kMapType = CU_TENSOR_MAP_DATA_TYPE_UINT8;  // (TMA copies bytes)
};
template <class T>
using OpT = typename Operand<T>::type;
template <class T>
using AccT = typename Operand<T>::Acc;
template <class T>
constexpr bool kInt8 = std::is_same_v<AccT<T>, int>;

// The score ||y||^2 - 2 <q, y> of a candidate from its norm s and cross term a: one fp32 fma, or exact in int32.
__device__ __forceinline__ float tile_score(float a, float s) { return fmaf(-2.0f, a, s); }
__device__ __forceinline__ int tile_score(int a, int s) { return s - 2 * a; }
// two adjacent staged accumulators or norms
template <class A>
using Pair = std::conditional_t<std::is_same_v<A, int>, int2, float2>;

// One K step of the cross terms of 64 query rows and TN candidates, D (+)= Ah Bh^T (+ Ah Bl^T + Al Bh^T for fp32).
template <class T, int TN>
__device__ __forceinline__ void cross_step(AccT<T> (&acc)[TN / 2], uint64_t ah, uint64_t al, uint64_t bh, uint64_t bl,
                                           uint32_t accumulate) {
  if constexpr (std::is_same_v<T, uint8_t>) {
    if constexpr (TN == 128) wgmma_u8(acc, ah, bh, accumulate);
    else wgmma_u8_n64(acc, ah, bh, accumulate);
  } else if constexpr (std::is_same_v<T, int8_t>) {
    if constexpr (TN == 128) wgmma_s8(acc, ah, bh, accumulate);
    else wgmma_s8_n64(acc, ah, bh, accumulate);
  } else if constexpr (std::is_same_v<T, __half>) {
    if constexpr (TN == 128) wgmma_f16(acc, ah, bh, accumulate);
    else wgmma_f16_n64(acc, ah, bh, accumulate);
  } else if constexpr (TN == 128) {
    wgmma_bf16(acc, ah, bh, accumulate);
    if constexpr (Operand<T>::kSplit) { wgmma_bf16(acc, ah, bl, 1u); wgmma_bf16(acc, al, bh, 1u); }
  } else {
    wgmma_bf16_n64(acc, ah, bh, accumulate);
    if constexpr (Operand<T>::kSplit) { wgmma_bf16_n64(acc, ah, bl, 1u); wgmma_bf16_n64(acc, al, bh, 1u); }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// column mean mu (fp32) of the fp32 values of X: fp64 sums over chunks of kMeanChunk rows, then over the chunks, in a
// fixed order (the same bits on every run)
// ---------------------------------------------------------------------------------------------------------------
constexpr int kMeanChunk = 512;
constexpr int kMaxGridY = 65535;

template <class T>
__global__ void __launch_bounds__(128)
knn_colsum_kernel(const T* __restrict__ X, int64_t n, int d, int chunks, double* __restrict__ part) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= d) return;
  for (int64_t ch = blockIdx.y; ch < chunks; ch += gridDim.y) {
    const int64_t r0 = ch * kMeanChunk;
    const int64_t r1 = r0 + kMeanChunk < n ? r0 + kMeanChunk : n;
    double s = 0.0;
    for (int64_t r = r0; r < r1; ++r) s += (double)elem_f32(X[r * d + c]);
    part[ch * d + c] = s;
  }
}

__global__ void __launch_bounds__(128)
knn_mean_kernel(const double* __restrict__ part, int chunks, int64_t n, int d, float* __restrict__ mu) {
  const int c = blockIdx.x * 128 + threadIdx.x;
  if (c >= d) return;
  double s = 0.0;
  for (int i = 0; i < chunks; ++i) s += part[(int64_t)i * d + c];
  mu[c] = (float)(s / (double)n);
}

// ---------------------------------------------------------------------------------------------------------------
// The error bound of the certificate (knn_certify_kernel).  s(y) = ||y^||^2 - 2 <q, y>~ is the score the tiles rank
// (fp32 norm and tensor-core cross term of the operand y^ = y - mu, or of y itself when the search is not centred),
// S(y) = ||q - y||^2 - ||q - mu||^2 its exact value.  |s(y) - S(y)| <= E(q) for every y, and the fp32 norm of the
// query lies within E(q) of ||q - mu||^2, with
//   E(q) = sigma (2 (a_cross |q^| M + eta (|q^| + M)) + a_norm M^2 + a_abs),   M^2 = max_y ||y^||^2 (fp32):
//   a_cross  the operand's rounding (bf16 x 3 split: the dropped lo x lo term and the split residual, 3.1 2^-16; a
//            centred value rounded to 16 bits: 2 eps + eps^2; an uncentred 16-bit element is its own exact operand: 0),
//            the centring's rounding (2.01 u, centred only), the fp32 accumulation of m products (2 u per addition,
//            u = 2^-24, allowing truncating tensor-core adds; m = 3 k_pad split, k_pad 16-bit) and the rounding of
//            the score's fma (u),
//   eta      fp16 subnormals of a centred operand: 2^-25 sqrt(k_pad) (an absolute error per element),
//   a_norm   the fp32 norm (ceil(k_pad / 32) + 8) u and the score's fma (u),
//   a_abs    underflow: 2^-126 per product and per square,
// and sigma = 2, a safety factor for second-order terms (tests/test_knn_offset_cpu.py derives the bound).
//
// 8-bit input.  The tiles rank by the exact score S(y), so the list holds the KK smallest exact distances and every
// row y it did not keep has D(y) = ||q - y||^2 >= D_KK = t + ||q||^2 (t: the worst kept score, exact).  The re-rank's
// value r(y) is an fp32 sum of d exact squared differences (each below 2^16, so exact in fp32) with at most
// L = ceil(d / 32) + 5 roundings on any path (the lane's fma chain, then five butterfly levels); a sum of non-negative
// terms so rounded lies within gamma = L u / (1 - L u) of its value, relatively, so r(y) >= (1 - gamma) D(y).  The row
// certifies when r_k < (1 - gamma) D_KK: no row outside the list can displace its k-th pair (ties fail and go to the
// direct search).  Every partial sum is an integer below 2^24, so exact, when d 255^2 <= 2^24 (d <= 258 for both
// 8-bit types): then gamma = 0 and the test is r_k < D_KK.  2^-50 covers the fp64 rounding of (1 - gamma) D_KK.
// tests/test_knn_int8_cpu.py derives gamma again and checks it against mde_dbg_knn8_gamma.
// ---------------------------------------------------------------------------------------------------------------
struct CertBound {
  double a_cen, a_unc;  // a_cross of the centred and of the uncentred operand
  double eta, a_norm, a_abs, delta;
  double gamma;         // 8-bit input: the re-rank's relative error bound
};
constexpr double kCertSafety = 2.0;

double knn8_gamma(int d) {
  if ((int64_t)d * 255 * 255 <= (1 << 24)) return 0.0;
  const double u = 0x1p-24, L = (double)((d + 31) / 32 + 5);
  return L * u / (1.0 - L * u) + 0x1p-50;
}

// d_max of an 8-bit type: the largest d for which every accumulator, norm and score of the tiles is exact in int32
// and every score stays below INT_MAX, the key of padded rows and empty list slots.  uint8: |2 <q, y>| <= 2 d 255^2
// and 0 <= ||y||^2 <= d 255^2, so 2 d 255^2 < 2^31 gives d <= 16 512.  int8: |<q, y>| <= d 128^2, so 2 <q, y> fits
// for d < 2^16, and the score ||y||^2 - 2 <q, y> <= d (128^2 + 2 128 127) = 48 896 d < 2^31 - 1 gives d <= 43 919.
template <class T>
constexpr int knn8_max_d() {
  if constexpr (std::is_same_v<T, uint8_t>) return (int)(((1ll << 31) - 1) / (2 * 255 * 255));
  else return (int)(((1ll << 31) - 2) / (128 * 128 + 2 * 128 * 127));
}
static_assert(knn8_max_d<uint8_t>() == 16512 && knn8_max_d<int8_t>() == 43919, "DESIGN section 11.9");

template <class T>
CertBound cert_bound(int d, int k_pad) {
  const double u = 0x1p-24;
  CertBound b{};
  if constexpr (kInt8<T>) {
    b.gamma = knn8_gamma(d);
    return b;
  }
  double op, op_unc = 0.0;
  int m = k_pad;
  if constexpr (Operand<T>::kSplit) { op = op_unc = 3.1 * 0x1p-16; m = 3 * k_pad; }
  else if constexpr (std::is_same_v<T, __half>) op = (2.0 + 0x1p-11) * 0x1p-11;
  else op = (2.0 + 0x1p-8) * 0x1p-8;
  b.a_cen = op + 2.01 * u + 2.0 * u * m + u;
  b.a_unc = op_unc + 2.0 * u * m + u;
  b.eta = std::is_same_v<T, __half> ? 0x1p-25 * sqrt((double)k_pad) : 0.0;
  b.a_norm = ((k_pad + 31) / 32 + 9) * u;
  b.a_abs = (2.0 * m + k_pad) * 0x1p-126 + (std::is_same_v<T, __half> ? 2.0 * k_pad * 0x1p-50 : 0.0);
  b.delta = ((d + 31) / 32 + 8) * u;
  return b;
}

// The search header in the workspace: uncertified row count, then maxima of squared norms as float bits
// (non-negative floats order as their bits; NaN orders above +inf) and the centring decision.
enum { kHdrCount, kHdrMaxNorm, kHdrMaxRaw, kHdrMaxCen, kHdrCentred, kHdrWords };

// ---------------------------------------------------------------------------------------------------------------
// norms: the largest fp32 squared norm of the raw rows and of the centred rows x - mu, for the centring decision
// ---------------------------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(256)
knn_maxnorm_kernel(const T* __restrict__ X, int64_t n, int d, const float* __restrict__ mu, unsigned* __restrict__ hdr) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  float raw = 0.0f, cen = 0.0f;
  for (int c = lane; c < d; c += 32) {
    const float x = elem_f32(X[row * d + c]), y = x - mu[c];
    raw = fmaf(x, x, raw);
    cen = fmaf(y, y, cen);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    raw += __shfl_xor_sync(kFull, raw, o);
    cen += __shfl_xor_sync(kFull, cen, o);
  }
  if (lane == 0) {
    atomicMax(hdr + kHdrMaxRaw, __float_as_uint(raw));
    atomicMax(hdr + kHdrMaxCen, __float_as_uint(cen));
  }
}

// Centre when the centred operand's cross-term bound, a_cen M_cen^2, is below the uncentred one, a_unc M_raw^2 (the
// same decision in every thread).  A 16-bit element is its own exact operand, while its centred value is rounded to
// 16 bits: data near the origin keeps X, data far from it is centred.
__device__ __forceinline__ bool knn_centre(const unsigned* hdr, const CertBound& b) {
  return b.a_cen * (double)__uint_as_float(hdr[kHdrMaxCen]) < b.a_unc * (double)__uint_as_float(hdr[kHdrMaxRaw]);
}

// ---------------------------------------------------------------------------------------------------------------
// prep: the operand (zero padded to n_pad x k_pad) of x^ = fl(x - mu), or of x itself when knn_centre says no: the
// bf16 hi / lo split of fp32 X, or x^ rounded to the 16-bit type of X (Xl unused; x itself when not centred, exact);
// squared norms of x^ (+inf on padded rows), the same arithmetic for every element type; their maximum over the rows
// to the header (+inf when an operand element is not finite, so that no row certifies)
// ---------------------------------------------------------------------------------------------------------------
// 8-bit input: X itself, zero padded, exact int32 squared norms and INT_MAX on padded rows (their score INT_MAX is
// never kept); mu, b and the header are not read.
template <class T>
__global__ void __launch_bounds__(256)
knn_prep_kernel(const T* __restrict__ X, int64_t n, int d, int64_t n_pad, int k_pad, const float* __restrict__ mu,
                CertBound b, OpT<T>* __restrict__ Xh, __nv_bfloat16* __restrict__ Xl, AccT<T>* __restrict__ norms,
                unsigned* __restrict__ hdr) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n_pad) return;
  if constexpr (kInt8<T>) {
    int acc = 0;
    for (int c = lane; c < k_pad; c += 32) {
      const T x = (row < n && c < d) ? X[row * d + c] : T(0);
      Xh[row * k_pad + c] = x;
      acc += (int)x * (int)x;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (lane == 0) norms[row] = (row < n) ? acc : INT_MAX;
    return;
  }
  const bool centre = knn_centre(hdr, b);
  if (row == 0 && lane == 0) hdr[kHdrCentred] = centre;
  float acc = 0.0f;
  bool bad = false;
  for (int c = lane; c < k_pad; c += 32) {
    const float x = (row < n && c < d) ? elem_f32(X[row * d + c]) - (centre ? mu[c] : 0.0f) : 0.0f;
    if constexpr (Operand<T>::kSplit) {
      const __nv_bfloat16 h = __float2bfloat16_rn(x);
      const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
      Xh[row * k_pad + c] = h;
      Xl[row * k_pad + c] = l;
    } else {
      const T o = T(x);  // round to nearest (fp16 overflows to inf beyond 65504); exact when not centred
      bad |= !isfinite(elem_f32(o));
      Xh[row * k_pad + c] = o;
    }
    acc += x * x;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
  bad = __any_sync(kFull, bad);
  if (lane == 0) {
    norms[row] = (row < n) ? acc : __int_as_float(0x7f800000);
    if (row < n) atomicMax(hdr + kHdrMaxNorm, bad ? 0x7f800000u : __float_as_uint(acc));
  }
}

// Replace the worst of the KK kept candidates by (dist, col) and find the new worst.  Static indices only, so the
// lists stay in registers.
template <class K>
__device__ __forceinline__ void keep_candidate(K (&bd)[kKK], int (&bi)[kKK], K dist, int col, K& thr, int& worst) {
#pragma unroll
  for (int q = 0; q < kKK; ++q) {
    if (q == worst) { bd[q] = dist; bi[q] = col; }
  }
  K m = bd[0]; int w = 0;
#pragma unroll
  for (int q = 1; q < kKK; ++q) { if (bd[q] > m) { m = bd[q]; w = q; } }
  thr = m; worst = w;
}

// ---------------------------------------------------------------------------------------------------------------
// tiles: tensor-core cross terms + running top-KK per query row
// ---------------------------------------------------------------------------------------------------------------
template <class T>
__global__ void __launch_bounds__(kThreads, 1)
knn_tile_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_l,
                const AccT<T>* __restrict__ norms, int64_t n, int64_t n_pad, int k_pad, QueryRange qr,
                int32_t* __restrict__ cand_idx, AccT<T>* __restrict__ cand_val) {
  using A = AccT<T>;
  constexpr int kBK = Operand<T>::kBlockK;
  extern __shared__ uint8_t smem_raw[];
  // carve: [stages x 64 KB, 1024-aligned] | staged accumulators [128][kAccStride] | norms[2][128] | barriers
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  A* s_acc = reinterpret_cast<A*>(gen + kStages * kStageBytes);
  A* s_norm = s_acc + kTileM * kAccStride;
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_norm + 2 * kTileN);
  const uint32_t bar0 = smem_u32(s_bar);
  // barriers: full[s] = bar0 + 8 s (TMA bytes landed), empty[s] = bar0 + 16 + 8 s (every consumer warp is done)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = k_pad / kBK;
  const int num_tiles = (int)(n_pad / kTileN);
  const int t_begin = qr.slice_begin(num_tiles), t_end = qr.slice_begin(num_tiles, 1);
  const int row0 = (int)qr.base + blockIdx.x * kTileM;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(bar0 + 8 * s, 1); mbar_init(bar0 + 16 + 8 * s, kConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===== TMA producer =====
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = t_begin; t < t_end; ++t) {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar0 + 16 + 8 * stage, phase ^ 1);  // slot released by the consumers
          const uint32_t full = bar0 + 8 * stage;
          const uint32_t dst = base + stage * kStageBytes;
          mbar_expect_tx(full, Operand<T>::kSplit ? kStageBytes : 2 * kOpBytes);  // 16/8-bit input: no lo parts
          tma_load_2d(dst, &map_h, kb * kBK, row0, full);
          if (Operand<T>::kSplit) tma_load_2d(dst + kOpBytes, &map_l, kb * kBK, row0, full);
          tma_load_2d(dst + 2 * kOpBytes, &map_h, kb * kBK, t * kTileN, full);
          if (Operand<T>::kSplit) tma_load_2d(dst + 3 * kOpBytes, &map_l, kb * kBK, t * kTileN, full);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns query rows row0 + 64 wg .. + 63 =====
  const int wg = warp >> 2;
  const int et = threadIdx.x & 127;            // thread within the warpgroup
  A* acc_s = s_acc + wg * 64 * kAccStride;
  A* sn = s_norm + wg * kTileN;
  // scan: two threads per query row, columns half, half + 2, half + 4, ...
  const int lrow = et >> 1, half = et & 1;
  const int row = row0 + wg * 64 + lrow;
  // accumulator fragment rows / columns of this thread (see wgmma_bf16)
  const int frow = 16 * (warp & 3) + (lane >> 2), fcol = 2 * (lane & 3);

  A bd[kKK];
  int bi[kKK];
#pragma unroll
  for (int q = 0; q < kKK; ++q) { bd[q] = key_inf<A>(); bi[q] = -1; }
  A thr = key_inf<A>();
  int worst = 0;
  A acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0;

  int stage = 0; uint32_t phase = 0;
  for (int t = t_begin; t < t_end; ++t) {
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(bar0 + 8 * stage, phase);  // operands landed
      const uint32_t sa = base + stage * kStageBytes;
      const uint64_t ah = smem_desc_sw128(sa + wg * 64 * kRowBytes), al = smem_desc_sw128(sa + kOpBytes + wg * 64 * kRowBytes);
      const uint64_t bh = smem_desc_sw128(sa + 2 * kOpBytes), bl = smem_desc_sw128(sa + 3 * kOpBytes);
#pragma unroll
      for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kKSteps; ++k) {
        const uint64_t adv = (uint64_t)((k * 32) >> 4);  // 32 bytes per K step inside the swizzle atom
        cross_step<T, kTileN>(acc, ah + adv, al + adv, bh + adv, bl + adv, (kb | k) != 0);
      }
      wgmma_commit();
      wgmma_wait_all();
#pragma unroll
      for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar0 + 16 + 8 * stage);  // this warp no longer reads the slot
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    // the previous tile's scan of acc_s / sn is finished by every thread of the warpgroup
    named_bar_sync(1 + wg, 128);
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      *reinterpret_cast<Pair<A>*>(acc_s + frow * kAccStride + 8 * j + fcol) = Pair<A>{acc[4 * j], acc[4 * j + 1]};
      *reinterpret_cast<Pair<A>*>(acc_s + (frow + 8) * kAccStride + 8 * j + fcol) = Pair<A>{acc[4 * j + 2], acc[4 * j + 3]};
    }
    sn[et] = __ldg(norms + (int64_t)t * kTileN + et);
    named_bar_sync(1 + wg, 128);
    const A* arow = acc_s + lrow * kAccStride;
#pragma unroll 4
    for (int i = 0; i < kTileN / 2; ++i) {
      const int c = 2 * i + half;
      const A dist = tile_score(arow[c], sn[c]);
      if (dist < thr) {
        const int col = t * kTileN + c;
        if (col != row) keep_candidate(bd, bi, dist, col, thr, worst);
      }
    }
  }
  // merge the two half-row lists: the odd-column thread hands its list to the even-column thread
  named_bar_sync(1 + wg, 128);
  A* xd = acc_s + lrow * kAccStride;
  int* xi = reinterpret_cast<int*>(xd + kKK);
  if (half) {
#pragma unroll
    for (int q = 0; q < kKK; ++q) { xd[q] = bd[q]; xi[q] = bi[q]; }
  }
  named_bar_sync(1 + wg, 128);
  if (!half) {
    for (int q = 0; q < kKK; ++q) {
      const A dist = xd[q];
      if (dist < thr) keep_candidate(bd, bi, dist, xi[q], thr, worst);
    }
    if (qr.has(row)) {
      const int64_t o = qr.list(row) * kKK;
#pragma unroll
      for (int q = 0; q < kKK; ++q) {
        cand_idx[o + q] = bi[q];
        cand_val[o + q] = bd[q];
      }
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// re-rank: exact fp32 squared distances of a row's candidates, the k smallest in ascending order
// (namespace mde, declared in mde_knn_select.cuh: mde_knn_approx.cu re-ranks its lists with the same kernels)
// ---------------------------------------------------------------------------------------------------------------
namespace mde {

template <class T>
__global__ void __launch_bounds__(256)
knn_rerank_kernel(const T* __restrict__ X, int64_t n, int d, const int32_t* __restrict__ cand_idx, int k,
                  int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int mine = cand_idx[row * kKK + lane];  // lane q owns candidate q
  float my_d = __int_as_float(0x7f800000);
  const T* xq = X + row * d;
  for (int q = 0; q < kKK; ++q) {
    const int c = __shfl_sync(kFull, mine, q);
    if (c < 0) continue;  // (warp-uniform)
    const T* xc = X + (int64_t)c * d;
    float acc = 0.0f;
    for (int j = lane; j < d; j += 32) { const float t = elem_f32(xq[j]) - elem_f32(xc[j]); acc = fmaf(t, t, acc); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (lane == q) my_d = acc;
  }
  // rank of (my_d, mine) among the 32 candidates: ties broken by index, missing candidates last
  int rank = 0;
  for (int q = 0; q < kKK; ++q) {
    const float od = __shfl_sync(kFull, my_d, q);
    const int oi = __shfl_sync(kFull, mine, q);
    if (q != lane && (od < my_d || (od == my_d && (unsigned)oi < (unsigned)mine))) ++rank;
  }
  if (rank < k) {
    out_idx[row * k + rank] = mine;
    out_d2[row * k + rank] = my_d;
  }
}

}  // namespace mde

namespace {

// ---------------------------------------------------------------------------------------------------------------
// wide tiles (k <= 64, KK = 96, TN = 128) and long tiles (k <= 256, KK = 288, TN = 64): as knn_tile_kernel for 64
// query rows, one running top-KK per row in shared memory, wgmma.m64n{TN}k16 on candidate tiles of TN rows
// ---------------------------------------------------------------------------------------------------------------
template <class T, int KK, int TN>
__global__ void __launch_bounds__(kWideThreads, 1)
knn_wide_tile_kernel(const __grid_constant__ CUtensorMap map_ah, const __grid_constant__ CUtensorMap map_al,
                     const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_l,
                     const AccT<T>* __restrict__ norms, int64_t n, int64_t n_pad, int k_pad, QueryRange qr,
                     int32_t* __restrict__ cand_idx, AccT<T>* __restrict__ cand_val) {
  static_assert(TN == 64 || TN == 128, "wgmma.m64n64 or m64n128");
  using A = AccT<T>;
  constexpr int kBK = Operand<T>::kBlockK;
  constexpr int kBOpBytes = TN * kRowBytes;
  constexpr int kStageB = kWideStageBytes<TN>;
  constexpr int kAccS = TN + 2;  // floats per staged accumulator row: the scan's float2 reads are conflict-free
  constexpr int kStride = WideList<KK>::kStride;
  extern __shared__ uint8_t smem_raw[];
  // carve: [stages x kStageB, 1024-aligned] | staged accumulators [64][kAccS] | norms[TN] |
  //        list distances [64][kStride] | list indices [64][kStride] | barriers
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  A* s_acc = reinterpret_cast<A*>(gen + kStages * kStageB);
  A* s_norm = s_acc + kWideTileM * kAccS;
  A* s_ld = s_norm + TN;
  int* s_li = reinterpret_cast<int*>(s_ld + kWideTileM * kStride);
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_li + kWideTileM * kStride);
  const uint32_t bar0 = smem_u32(s_bar);
  // barriers: full[s] = bar0 + 8 s (TMA bytes landed), empty[s] = bar0 + 16 + 8 s (every consumer warp is done)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = k_pad / kBK;
  const int num_tiles = (int)(n_pad / TN);
  const int t_begin = qr.slice_begin(num_tiles), t_end = qr.slice_begin(num_tiles, 1);
  const int row0 = (int)qr.base + blockIdx.x * kWideTileM;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(bar0 + 8 * s, 1); mbar_init(bar0 + 16 + 8 * s, kWideConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kWideConsumerWarps) {
    // ===== TMA producer =====
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = t_begin; t < t_end; ++t) {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar0 + 16 + 8 * stage, phase ^ 1);  // slot released by the consumers
          const uint32_t full = bar0 + 8 * stage;
          const uint32_t dst = base + stage * kStageB;
          mbar_expect_tx(full, Operand<T>::kSplit ? kStageB : kAOpBytes + kBOpBytes);  // 16/8-bit input: no lo parts
          tma_load_2d(dst, &map_ah, kb * kBK, row0, full);
          if (Operand<T>::kSplit) tma_load_2d(dst + kAOpBytes, &map_al, kb * kBK, row0, full);
          tma_load_2d(dst + 2 * kAOpBytes, &map_h, kb * kBK, t * TN, full);
          if (Operand<T>::kSplit) tma_load_2d(dst + 2 * kAOpBytes + kBOpBytes, &map_l, kb * kBK, t * TN, full);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumers: the warpgroup owns query rows row0 .. row0 + 63, two adjacent lanes per row =====
  const int et = threadIdx.x;
  const int lrow = et >> 1, half = et & 1;
  const int row = row0 + lrow;
  const int frow = 16 * warp + (lane >> 2), fcol = 2 * (lane & 3);
  WideList<KK, A> list;
  list.init(s_ld + lrow * kStride, s_li + lrow * kStride, half);
  A acc[TN / 2];
#pragma unroll
  for (int i = 0; i < TN / 2; ++i) acc[i] = 0;

  int stage = 0; uint32_t phase = 0;
  for (int t = t_begin; t < t_end; ++t) {
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(bar0 + 8 * stage, phase);  // operands landed
      const uint32_t sa = base + stage * kStageB;
      const uint64_t ah = smem_desc_sw128(sa), al = smem_desc_sw128(sa + kAOpBytes);
      const uint64_t bh = smem_desc_sw128(sa + 2 * kAOpBytes), bl = smem_desc_sw128(sa + 2 * kAOpBytes + kBOpBytes);
#pragma unroll
      for (int i = 0; i < TN / 2; ++i) fence_operand(acc[i]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kKSteps; ++k) {
        const uint64_t adv = (uint64_t)((k * 32) >> 4);
        cross_step<T, TN>(acc, ah + adv, al + adv, bh + adv, bl + adv, (kb | k) != 0);
      }
      wgmma_commit();
      wgmma_wait_all();
#pragma unroll
      for (int i = 0; i < TN / 2; ++i) fence_operand(acc[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar0 + 16 + 8 * stage);  // this warp no longer reads the slot
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    // the previous tile's scan of s_acc / s_norm is finished by every consumer thread
    named_bar_sync(1, 128);
#pragma unroll
    for (int j = 0; j < TN / 8; ++j) {
      *reinterpret_cast<Pair<A>*>(s_acc + frow * kAccS + 8 * j + fcol) = Pair<A>{acc[4 * j], acc[4 * j + 1]};
      *reinterpret_cast<Pair<A>*>(s_acc + (frow + 8) * kAccS + 8 * j + fcol) = Pair<A>{acc[4 * j + 2], acc[4 * j + 3]};
    }
    if (et < TN) s_norm[et] = __ldg(norms + (int64_t)t * TN + et);
    named_bar_sync(1, 128);
    // both lanes of the row offer every column, in column order
    const Pair<A>* arow = reinterpret_cast<const Pair<A>*>(s_acc + lrow * kAccS);
    const Pair<A>* sn = reinterpret_cast<const Pair<A>*>(s_norm);
#pragma unroll 2
    for (int i = 0; i < TN / 2; ++i) {
      const Pair<A> a = arow[i], s = sn[i];
      const int col = t * TN + 2 * i;
      if (col != row && col < n) list.offer(tile_score(a.x, s.x), col);
      if (col + 1 != row && col + 1 < n) list.offer(tile_score(a.y, s.y), col + 1);
    }
  }
  if (qr.has(row)) list.store(cand_idx + qr.list(row) * KK, cand_val + qr.list(row) * KK);
}

}  // namespace

namespace mde {

// Exact fp32 squared distances of a row's KK candidates (the arithmetic of knn_rerank_kernel), the k smallest in
// ascending order; lane q owns candidates q, q + 32, q + 64, ..., ranks are taken over all KK.  Row r of the n lists
// and of the output is row lo + r of X.
template <class T, int KK>
__device__ __forceinline__ void wide_rerank_row(const T* __restrict__ X, int64_t lo, int64_t n, int d,
                                                const int32_t* __restrict__ cand_idx, int k,
                                                int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  constexpr int kPer = KK / 32;
  int mine[kPer];
  float my_d[kPer];
  const T* xq = X + (lo + row) * d;
#pragma unroll
  for (int s = 0; s < kPer; ++s) {
    mine[s] = cand_idx[row * KK + 32 * s + lane];
    my_d[s] = __int_as_float(0x7f800000);
    for (int q = 0; q < 32; ++q) {
      const int c = __shfl_sync(kFull, mine[s], q);
      if (c < 0) continue;  // (warp-uniform)
      const T* xc = X + (int64_t)c * d;
      float acc = 0.0f;
      for (int j = lane; j < d; j += 32) { const float t = elem_f32(xq[j]) - elem_f32(xc[j]); acc = fmaf(t, t, acc); }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
      if (lane == q) my_d[s] = acc;
    }
  }
  // rank of each owned (distance, index) among the KK: ties broken by index, missing candidates last
  int rank[kPer] = {};
#pragma unroll
  for (int s2 = 0; s2 < kPer; ++s2) {
    for (int q = 0; q < 32; ++q) {
      const float od = __shfl_sync(kFull, my_d[s2], q);
      const int oi = __shfl_sync(kFull, mine[s2], q);
#pragma unroll
      for (int s = 0; s < kPer; ++s) {
        if ((q != lane || s2 != s) && (od < my_d[s] || (od == my_d[s] && (unsigned)oi < (unsigned)mine[s]))) ++rank[s];
      }
    }
  }
#pragma unroll
  for (int s = 0; s < kPer; ++s) {
    if (rank[s] < k) {
      out_idx[row * k + rank[s]] = mine[s];
      out_d2[row * k + rank[s]] = my_d[s];
    }
  }
}

template <class T>
__global__ void __launch_bounds__(256)
knn_wide_rerank_kernel(const T* __restrict__ X, int64_t n, int d, const int32_t* __restrict__ cand_idx, int k,
                       int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  wide_rerank_row<T, kWideKK>(X, 0, n, d, cand_idx, k, out_idx, out_d2);
}

// the 288 candidates of the long search, with the same arithmetic, for the n query rows lo .. lo + n - 1 of X
// (lo = 0 but for the long row search)
template <class T>
__global__ void __launch_bounds__(256)
knn_long_rerank_kernel(const T* __restrict__ X, int64_t lo, int64_t n, int d, const int32_t* __restrict__ cand_idx,
                       int k, int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  wide_rerank_row<T, kLongKK>(X, lo, n, d, cand_idx, k, out_idx, out_d2);
}

template <class T>
int knn_dense_rerank(int kk, const T* X, int64_t n, int d, const int32_t* cand_idx, int k, int32_t* out_idx,
                     float* out_d2, cudaStream_t st) {
  const unsigned grid = (unsigned)((n + 7) / 8);
  if (kk == kNarrowKK) knn_rerank_kernel<T><<<grid, 256, 0, st>>>(X, n, d, cand_idx, k, out_idx, out_d2);
  else if (kk == kWideKK) knn_wide_rerank_kernel<T><<<grid, 256, 0, st>>>(X, n, d, cand_idx, k, out_idx, out_d2);
  else if (kk == kLongKK) knn_long_rerank_kernel<T><<<grid, 256, 0, st>>>(X, 0, n, d, cand_idx, k, out_idx, out_d2);
  else return MDE_E_INVALID;
  MDE_LAUNCH_CHECK();
  return 0;
}
template int knn_dense_rerank<float>(int, const float*, int64_t, int, const int32_t*, int, int32_t*, float*,
                                     cudaStream_t);
template int knn_dense_rerank<__half>(int, const __half*, int64_t, int, const int32_t*, int, int32_t*, float*,
                                      cudaStream_t);
template int knn_dense_rerank<__nv_bfloat16>(int, const __nv_bfloat16*, int64_t, int, const int32_t*, int, int32_t*,
                                             float*, cudaStream_t);
template int knn_dense_rerank<uint8_t>(int, const uint8_t*, int64_t, int, const int32_t*, int, int32_t*, float*,
                                       cudaStream_t);
template int knn_dense_rerank<int8_t>(int, const int8_t*, int64_t, int, const int32_t*, int, int32_t*, float*,
                                      cudaStream_t);

}  // namespace mde

namespace {

// ---------------------------------------------------------------------------------------------------------------
// merge: the re-rank of a row searched in S candidate slices (or of a query range that does not start at row 0).
// One warp per query row r (global row lo + r) computes the exact fp32 distances of its S KK candidates with the
// re-rank's arithmetic (the same bits), stages them in shared memory and writes the k smallest (distance, index)
// pairs, ascending, to row r of the compact output; missing candidates (-1) order last, as in the re-rank.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kMergeWarps = 4;

template <class T>
__global__ void __launch_bounds__(kMergeWarps * 32)
knn_merge_rerank_kernel(const T* __restrict__ X, int d, int64_t lo, int64_t rows,
                        const int32_t* __restrict__ cand_idx, int cands, int k, int32_t* __restrict__ out_idx,
                        float* __restrict__ out_d2) {
  extern __shared__ float s_merge[];  // per warp: distances [cands], indices [cands]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * kMergeWarps + warp;
  if (r >= rows) return;
  float* sd = s_merge + (size_t)warp * 2 * cands;
  unsigned* si = reinterpret_cast<unsigned*>(sd + cands);
  const T* xq = X + (lo + r) * d;
  for (int b = 0; b < cands; b += 32) {
    const int mine = cand_idx[r * cands + b + lane];
    float my_d = __int_as_float(0x7f800000);
    for (int q = 0; q < 32; ++q) {
      const int c = __shfl_sync(kFull, mine, q);
      if (c < 0) continue;  // (warp-uniform)
      const T* xc = X + (int64_t)c * d;
      float acc = 0.0f;
      for (int j = lane; j < d; j += 32) { const float t = elem_f32(xq[j]) - elem_f32(xc[j]); acc = fmaf(t, t, acc); }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
      if (lane == q) my_d = acc;
    }
    sd[b + lane] = my_d;
    si[b + lane] = (unsigned)mine;
  }
  __syncwarp();
  // rank of each candidate among the S KK: ties broken by index (slices hold disjoint rows), missing candidates last
  for (int j = lane; j < cands; j += 32) {
    const float dj = sd[j];
    const unsigned ij = si[j];
    int rank = 0;
    for (int q = 0; q < cands; ++q) rank += (sd[q] < dj || (sd[q] == dj && si[q] < ij));
    if (rank < k) {
      out_idx[r * k + rank] = (int32_t)ij;
      out_d2[r * k + rank] = dj;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// long merge: the candidates of a row searched in S candidate slices by the long tiles (mde_knn_long_rows; DESIGN
// section 11.8).  Slice y keeps the 288 smallest (score, index) pairs of its candidates in WideList's order (-0 == +0,
// ties by index, an empty slot as (key_inf, INT_MAX)), a strict total order, so the kept set does not depend on the
// order of the offers.  Every member of the full search's 288 is among its own slice's 288, so the 288 smallest of
// the S 288 pairs in the same order are exactly the full search's candidates, and their worst score is the full
// search's worst kept score.  Ranking S 288 <= 4 608 pairs against each other would cost 21 M comparisons per row, so
// one CTA per row radix-selects them instead: each pair becomes the 64-bit key (order-preserving bits of the score,
// index; an empty slot's -1 as 0xffffffff), the keys stay in registers (18 per thread at S = 16), and an MSB-first
// select over 8-bit digits narrows the prefix of the 288-th key, stopping at the first digit whose bin holds exactly
// the keys still needed.  Shared memory: a 256-bin histogram and four control words.  The pairs below the prefix, then
// enough pairs equal to it (only ever identical empty slots), are copied, as the tiles wrote them, to sel[r][.]; their
// order there is free (the re-rank ranks all 288 and the certificate takes their maximum).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kSelThreads = 256;
constexpr int kSelPer = kMaxSlices * kLongKK / kSelThreads;  // keys per thread at S = kMaxSlices
static_assert(kMaxSlices * kLongKK % kSelThreads == 0, "whole keys per thread");

// order-preserving unsigned bits of a tile score: -0 and +0 map to the same key
__device__ __forceinline__ uint32_t score_bits(float v) {
  uint32_t b = __float_as_uint(v);
  if (b == 0x80000000u) b = 0u;
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ uint32_t score_bits(int v) { return (uint32_t)v ^ 0x80000000u; }

template <class A>
__global__ void __launch_bounds__(kSelThreads)
knn_long_select_kernel(const int32_t* __restrict__ cand_idx, const A* __restrict__ cand_val, int slices,
                       int32_t* __restrict__ sel, A* __restrict__ sel_val) {
  __shared__ unsigned s_hist[256];
  __shared__ unsigned s_ctl[4];  // bin of the 288-th key, keys still needed, count of that bin | output counters
  const int tid = threadIdx.x, lane = tid & 31;
  const int64_t r = blockIdx.x;
  const int cands = slices * kLongKK;
  const int32_t* ri = cand_idx + r * cands;
  const A* rv = cand_val + r * cands;
  uint64_t key[kSelPer];
#pragma unroll
  for (int j = 0; j < kSelPer; ++j) {
    const int c = tid + j * kSelThreads;
    key[j] = c < cands ? ((uint64_t)score_bits(rv[c]) << 32) | (uint32_t)ri[c] : ~0ull;
  }
  uint64_t prefix = 0, mask = 0;
  unsigned need = kLongKK;  // of the keys that match the prefix
  for (int shift = 56; shift >= 0; shift -= 8) {
    s_hist[tid] = 0u;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kSelPer; ++j) {
      const bool in = tid + j * kSelThreads < cands && (key[j] & mask) == prefix;
      const unsigned bin = in ? (unsigned)(key[j] >> shift) & 255u : 256u;
      const unsigned peers = __match_any_sync(kFull, bin);  // one shared-memory atomic per bin and warp
      if (in && lane == __ffs(peers) - 1) atomicAdd(&s_hist[bin], (unsigned)__popc(peers));
    }
    __syncthreads();
    if (tid < 32) {
      // lane l scans bins 8 l .. 8 l + 7; the lane whose range holds the need-th key finds its bin
      unsigned h[8], sum = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) { h[b] = s_hist[8 * lane + b]; sum += h[b]; }
      unsigned incl = sum;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const unsigned v = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += v;
      }
      unsigned below = incl - sum;
      if (below < need && need <= incl) {
        int b = 0;
        while (below + h[b] < need) below += h[b++];
        s_ctl[0] = 8 * lane + b; s_ctl[1] = need - below; s_ctl[2] = h[b];
      }
    }
    __syncthreads();
    prefix |= (uint64_t)s_ctl[0] << shift;
    mask |= 0xffull << shift;
    need = s_ctl[1];
    const bool done = s_ctl[2] == need;  // the bin holds exactly the keys still needed
    __syncthreads();                      // (s_ctl and s_hist are rewritten below)
    if (done) break;
  }
  // kLongKK - need keys lie below the prefix; `need` more match it
  if (tid == 0) { s_ctl[2] = 0u; s_ctl[3] = 0u; }
  __syncthreads();
  int32_t* so = sel + r * kLongKK;
  A* vo = sel_val + r * kLongKK;
#pragma unroll
  for (int j = 0; j < kSelPer; ++j) {
    const int c = tid + j * kSelThreads;
    if (c >= cands) continue;
    const uint64_t m = key[j] & mask;
    int o = -1;
    if (m < prefix) {
      o = (int)atomicAdd(&s_ctl[2], 1u);
    } else if (m == prefix) {
      const unsigned t = atomicAdd(&s_ctl[3], 1u);
      if (t < need) o = (int)(kLongKK - need + t);
    }
    if (o >= 0) { so[o] = ri[c]; vo[o] = rv[c]; }
  }
}

}  // namespace

namespace {

// ---------------------------------------------------------------------------------------------------------------
// certificate: is the re-ranked list of a row the k smallest (distance, index) over ALL rows?
//
// Every row the tiles did not keep scored at least t, the worst kept score (+inf when the list was never filled:
// every row was kept); a row searched in S candidate slices takes the smallest of the S slices' worst kept scores,
// since every row a slice did not keep scored at least that slice's worst.  With the bound E(q) above (cert_bound), a row that was not kept lies at an exact distance of at
// least t - E(q) + ||q^||^2 - E(q); when that exceeds d2_k (1 + delta) / (1 - delta), where d2_k is the k-th
// re-ranked fp32 distance and delta bounds the re-rank's relative rounding, its fp32 distance exceeds d2_k and it
// cannot enter the list.  A row that fails is searched directly (knn_direct_kernel); a false failure costs time
// only.  The uncertified rows are appended to rows[] (in no particular order: each is searched on its own) and
// counted in the header.  8-bit input (A = int): t is exact, and the row certifies when d2_k < (1 - gamma) (t +
// ||q||^2) (cert_bound), or when t = INT_MAX (no list was ever full: every row was kept).
// ---------------------------------------------------------------------------------------------------------------
template <class A>
__global__ void __launch_bounds__(256)
knn_certify_kernel(const A* __restrict__ cand_val, int kk, int slices, const A* __restrict__ norms,
                   const float* __restrict__ d2_out, int k, int64_t lo, int64_t n, CertBound b,
                   unsigned* __restrict__ hdr, int32_t* __restrict__ rows) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // of the query range
  if (row >= n) return;
  const A* cv = cand_val + row * slices * kk;
  if constexpr (std::is_same_v<A, int>) {
    int t = INT_MAX;
    for (int s = 0; s < slices; ++s, cv += kk) {
      int ts = INT_MIN;
      for (int q = lane; q < kk; q += 32) ts = max(ts, cv[q]);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ts = max(ts, __shfl_xor_sync(kFull, ts, o));
      t = min(t, ts);
    }
    if (lane || t == INT_MAX) return;
    const double D = (double)((int64_t)t + norms[lo + row]);
    if (!((double)d2_out[row * k + k - 1] < (1.0 - b.gamma) * D))
      rows[atomicAdd(reinterpret_cast<int*>(hdr + kHdrCount), 1)] = (int32_t)row;
    return;
  }
  float t = __int_as_float(0x7f800000);
  for (int s = 0; s < slices; ++s, cv += kk) {
    float ts = -__int_as_float(0x7f800000);
    for (int q = lane; q < kk; q += 32) ts = fmaxf(ts, cv[q]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ts = fmaxf(ts, __shfl_xor_sync(kFull, ts, o));
    t = fminf(t, ts);
  }
  if (lane) return;
  const bool centred = hdr[kHdrCentred] != 0;
  const double a_cross = centred ? b.a_cen : b.a_unc, eta = centred ? b.eta : 0.0;
  const double M2 = (double)__uint_as_float(hdr[kHdrMaxNorm]), M = sqrt(M2);
  const double qn = (double)norms[lo + row], qa = sqrt(qn);
  const double E = kCertSafety * (2.0 * (a_cross * qa * M + eta * (qa + M)) + b.a_norm * M2 + b.a_abs);
  const double lhs = (double)d2_out[row * k + k - 1] * (1.0 + b.delta) / (1.0 - b.delta) - qn + E;
  if (!(lhs < (double)t - E)) rows[atomicAdd(reinterpret_cast<int*>(hdr + kHdrCount), 1)] = (int32_t)row;
}

// ---------------------------------------------------------------------------------------------------------------
// direct search of the uncertified rows (row r of the query range is row lo + r of X): one warp per row sweeps all n
// rows with the re-rank's arithmetic (the same fp32 bits) and keeps the k smallest (distance, index) pairs, ascending.  Only pairs up to the re-rank's k-th pair
// can belong (the re-rank's k rows are k candidates with these very distances), which keeps insertions rare.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool pair_before(float d1, unsigned i1, float d2, unsigned i2) {
  return d1 < d2 || (d1 == d2 && i1 < i2);
}

template <class T>
__global__ void __launch_bounds__(256)
knn_direct_kernel(const T* __restrict__ X, int64_t n, int d, int k, int64_t lo, const unsigned* __restrict__ hdr,
                  const int32_t* __restrict__ rows, int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  __shared__ float s_d[8][kLongMaxK];
  __shared__ unsigned s_i[8][kLongMaxK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t slot = (int64_t)blockIdx.x * 8 + warp;
  if (slot >= (int64_t)hdr[kHdrCount]) return;
  const int64_t row = rows[slot];
  float* ld = s_d[warp];
  unsigned* li = s_i[warp];
  for (int j = lane; j < k; j += 32) { ld[j] = __int_as_float(0x7f800000); li[j] = 0xffffffffu; }
  __syncwarp();
  const float bd = out_d2[row * k + k - 1];
  const unsigned bi = (unsigned)out_idx[row * k + k - 1];
  float thr = __int_as_float(0x7f800000);
  unsigned thi = 0xffffffffu;
  int worst = 0;
  const T* xq = X + (lo + row) * d;
  for (int64_t c = 0; c < n; ++c) {
    if (c == lo + row) continue;
    const T* xc = X + c * d;
    float acc = 0.0f;
    for (int j = lane; j < d; j += 32) { const float t = elem_f32(xq[j]) - elem_f32(xc[j]); acc = fmaf(t, t, acc); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    // (warp-uniform) at most the re-rank's k-th pair, and before the worst kept pair
    if (pair_before(bd, bi, acc, (unsigned)c) || !pair_before(acc, (unsigned)c, thr, thi)) continue;
    if (lane == 0) { ld[worst] = acc; li[worst] = (unsigned)c; }
    __syncwarp();
    // the new worst: the largest (distance, index, slot) of the list
    float m = -__int_as_float(0x7f800000); unsigned mi = 0; int w = -1;
    for (int j = lane; j < k; j += 32) {
      if (pair_before(m, mi, ld[j], li[j]) || (m == ld[j] && mi == li[j])) { m = ld[j]; mi = li[j]; w = j; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(kFull, m, o);
      const unsigned omi = __shfl_xor_sync(kFull, mi, o);
      const int ow = __shfl_xor_sync(kFull, w, o);
      if (pair_before(m, mi, om, omi) || (m == om && mi == omi && ow > w)) { m = om; mi = omi; w = ow; }
    }
    thr = m; thi = mi; worst = w;
    __syncwarp();
  }
  // ascending by (distance, index): the rank of every slot among the k
  int rank[kLongMaxK / 32];
#pragma unroll
  for (int s = 0; s < kLongMaxK / 32; ++s) {
    const int j = lane + 32 * s;
    rank[s] = 0;
    if (j < k) for (int q = 0; q < k; ++q) rank[s] += pair_before(ld[q], li[q], ld[j], li[j]);
  }
#pragma unroll
  for (int s = 0; s < kLongMaxK / 32; ++s) {
    const int j = lane + 32 * s;
    if (j < k) {
      out_idx[row * k + rank[s]] = (int32_t)li[j];
      out_d2[row * k + rank[s]] = ld[j];
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// cuTensorMapEncodeTiled, fetched once through the runtime (no link-time libcuda dependency)
int tensor_map_encoder(EncodeTiledFn* out) {
  static EncodeTiledFn enc = nullptr;
  if (!enc) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    MDE_CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) return MDE_E_UNSUPPORTED;
    enc = (EncodeTiledFn)fn;
  }
  *out = enc;
  return 0;
}

// Tensor map of an n_pad x k_pad 16-bit (bf16, fp16) or 8-bit operand, loaded in boxes of box_rows x 128 bytes
// (128-byte swizzle).
int make_map(EncodeTiledFn enc, CUtensorMap* map, void* ptr, int64_t n_pad, int k_pad, int box_rows = kTileM,
             CUtensorMapDataType type = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  const int elem = type == CU_TENSOR_MAP_DATA_TYPE_UINT8 ? 1 : 2;
  const cuuint64_t dims[2] = {(cuuint64_t)k_pad, (cuuint64_t)n_pad};
  const cuuint64_t strides[1] = {(cuuint64_t)k_pad * elem};
  const cuuint32_t box[2] = {(cuuint32_t)(kRowBytes / elem), (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, type, 2, ptr, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : MDE_E_INVALID;
}

struct KnnLayout {
  int64_t n_pad; int k_pad, chunks, slices;
  size_t off_h, off_l, off_norm, off_ci, off_cv, off_sel, off_selv, off_mu, off_part, off_hdr, off_rows, total;
};

// The tile shape of a search: tm query rows per CTA, tn candidates per tile, kk candidates kept per row (kKK, kWideKK
// for the wide search, kLongKK for the long one); split: whether the candidate sweep may be split into slices.
struct Shape { int tm, tn, kk; bool split; };
constexpr Shape kNarrow{kTileM, kTileN, kKK, true}, kWide{kWideTileM, kTileN, kWideKK, true};
// The full long searches keep one slice (their query tiles fill the SMs from n = 8 448 on, and their bits, fallback
// counts and times stay those of the one-slice sweep); the long row search splits and merges (knn_long_select_kernel).
constexpr Shape kLong{kWideTileM, kLongTileN, kLongKK, false}, kLongRows{kWideTileM, kLongTileN, kLongKK, true};

// Candidate slices of a search of `rows` query rows against the n rows of X (mde_logic.h: knn_slices).
int search_slices(int64_t n, int64_t rows, Shape sh) {
  if (!sh.split) return 1;
  const int64_t n_pad = (n + kTileN - 1) / kTileN * kTileN;
  return knn_slices((rows + sh.tm - 1) / sh.tm, n_pad / sh.tn, kNumSMs, kMaxSlices);
}

// The operand of an element type: the bf16 hi / lo split of fp32 input, a 16-bit operand (no lo part: off_l == off_h,
// 2 n_pad k_pad bytes fewer), or an 8-bit one (1 byte per element, k_pad a multiple of 128, and no centring: no column
// mean or its sums).
enum OpKind { kOpSplit, kOp16, kOp8 };
template <class T>
constexpr OpKind kOpKind = kInt8<T> ? kOp8 : Operand<T>::kSplit ? kOpSplit : kOp16;

// rows: query rows of the search (n for a full one), each with one list of sh.kk candidates per slice
KnnLayout knn_layout(int64_t n, int d, int64_t rows, Shape sh, OpKind op) {
  KnnLayout L;
  const int elem = op == kOp8 ? 1 : 2, block_k = kRowBytes / elem;
  const bool split = op == kOpSplit, centring = op != kOp8;
  L.n_pad = (n + kTileN - 1) / kTileN * kTileN;
  L.k_pad = (d + block_k - 1) / block_k * block_k;
  L.chunks = centring ? (int)((n + kMeanChunk - 1) / kMeanChunk) : 0;
  L.slices = search_slices(n, rows, sh);
  // room for the lists of rows x S query rows: rows itself, or, when the rule may split, the most a split can hold
  // (q_tiles S <= kNumSMs, S <= kMaxSlices).  Monotone in rows: a workspace sized for a search fits every smaller one.
  int64_t cap = rows;
  if (sh.split) {
    const int64_t split = rows * kMaxSlices < (int64_t)kNumSMs * sh.tm ? rows * kMaxSlices : (int64_t)kNumSMs * sh.tm;
    if (split > cap) cap = split;
  }
  const size_t lists = (size_t)cap * sh.kk;
  // the long row search's merged lists: one list of kLongKK per query row (knn_long_select_kernel)
  const size_t merged = sh.split && sh.kk == kLongKK ? (size_t)rows * kLongKK : 0;
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  size_t o = 0;
  L.off_h = o; o = up(o + (size_t)L.n_pad * L.k_pad * elem);
  L.off_l = split ? o : L.off_h;
  if (split) o = up(o + (size_t)L.n_pad * L.k_pad * 2);
  L.off_norm = o; o = up(o + (size_t)L.n_pad * 4);
  L.off_ci = o; o = up(o + lists * 4);
  L.off_cv = o; o = up(o + lists * 4);
  L.off_sel = o; o = up(o + merged * 4);
  L.off_selv = o; o = up(o + merged * 4);
  L.off_mu = o; o = up(o + (centring ? (size_t)d * 4 : 0));  // column mean
  L.off_part = o; o = up(o + (size_t)L.chunks * d * 8);      // its per-chunk fp64 sums
  L.off_hdr = o; o = up(o + 4 * kHdrWords);                  // the search header (kHdr*)
  L.off_rows = o; o = up(o + (size_t)rows * 4);              // the uncertified rows
  L.total = o;
  return L;
}

// The tiles' operand and norms: column mean, the centring decision, then prep.
template <class T>
int centre_and_prep(const T* X, int64_t n, int d, const KnnLayout& L, uint8_t* w, cudaStream_t st) {
  double* part = reinterpret_cast<double*>(w + L.off_part);
  float* mu = reinterpret_cast<float*>(w + L.off_mu);
  unsigned* hdr = reinterpret_cast<unsigned*>(w + L.off_hdr);
  MDE_CUDA_TRY(cudaMemsetAsync(hdr, 0, 4 * kHdrWords, st));
  if constexpr (!kInt8<T>) {  // an 8-bit operand is exact wherever the data sits: no centring
    const unsigned gy = (unsigned)(L.chunks < kMaxGridY ? L.chunks : kMaxGridY);
    knn_colsum_kernel<T><<<dim3((unsigned)((d + 127) / 128), gy), 128, 0, st>>>(X, n, d, L.chunks, part);
    MDE_LAUNCH_CHECK();
    knn_mean_kernel<<<(unsigned)((d + 127) / 128), 128, 0, st>>>(part, L.chunks, n, d, mu);
    MDE_LAUNCH_CHECK();
    knn_maxnorm_kernel<T><<<(unsigned)((n + 7) / 8), 256, 0, st>>>(X, n, d, mu, hdr);
    MDE_LAUNCH_CHECK();
  }
  knn_prep_kernel<T><<<(unsigned)((L.n_pad + 7) / 8), 256, 0, st>>>(
      X, n, d, L.n_pad, L.k_pad, mu, cert_bound<T>(d, L.k_pad), reinterpret_cast<OpT<T>*>(w + L.off_h),
      reinterpret_cast<__nv_bfloat16*>(w + L.off_l), reinterpret_cast<AccT<T>*>(w + L.off_norm), hdr);
  MDE_LAUNCH_CHECK();
  return 0;
}

// After the tiles: re-rank the candidates of every query row (rows lo .. hi - 1 of X; the S KK of a sliced search
// are merged: by an exact re-rank of all S KK for the narrow and wide searches, by selecting the full search's 288
// before the long re-rank for the long one), certify every row, search the uncertified rows directly; with `fallback_rows`, wait for the stream
// and report how many rows that was.  Outputs are compact: row r holds row lo + r of X.
template <class T>
int rerank_certify(int kk, const T* X, int64_t n, int d, int64_t lo, int64_t hi, int k, int32_t* idx_out,
                   float* d2_out, const KnnLayout& L, uint8_t* w, cudaStream_t st, int* fallback_rows) {
  using A = AccT<T>;
  const int64_t rows = hi - lo;
  const int32_t* ci = reinterpret_cast<const int32_t*>(w + L.off_ci);
  const A* cv = reinterpret_cast<const A*>(w + L.off_cv);
  int slices = L.slices, rc;
  if (kk == kLongKK) {
    if (slices > 1) {  // the full search's 288 candidates of each row, from its S lists
      int32_t* sel = reinterpret_cast<int32_t*>(w + L.off_sel);
      A* selv = reinterpret_cast<A*>(w + L.off_selv);
      knn_long_select_kernel<A><<<(unsigned)rows, kSelThreads, 0, st>>>(ci, cv, slices, sel, selv);
      MDE_LAUNCH_CHECK();
      ci = sel; cv = selv; slices = 1;
    }
    knn_long_rerank_kernel<T><<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(X, lo, rows, d, ci, k, idx_out, d2_out);
    MDE_LAUNCH_CHECK();
  } else if (L.slices == 1 && lo == 0) {
    if ((rc = knn_dense_rerank<T>(kk, X, rows, d, ci, k, idx_out, d2_out, st))) return rc;
  } else {
    const int cands = L.slices * kk;
    knn_merge_rerank_kernel<T><<<(unsigned)((rows + kMergeWarps - 1) / kMergeWarps), kMergeWarps * 32,
                                 (size_t)kMergeWarps * cands * 8, st>>>(X, d, lo, rows, ci, cands, k, idx_out, d2_out);
    MDE_LAUNCH_CHECK();
  }
  unsigned* hdr = reinterpret_cast<unsigned*>(w + L.off_hdr);
  int32_t* uncert = reinterpret_cast<int32_t*>(w + L.off_rows);
  const unsigned grid = (unsigned)((rows + 7) / 8);
  knn_certify_kernel<A><<<grid, 256, 0, st>>>(cv, kk, slices, reinterpret_cast<const A*>(w + L.off_norm), d2_out, k,
                                             lo, rows, cert_bound<T>(d, L.k_pad), hdr, uncert);
  MDE_LAUNCH_CHECK();
  knn_direct_kernel<T><<<grid, 256, 0, st>>>(X, n, d, k, lo, hdr, uncert, idx_out, d2_out);
  MDE_LAUNCH_CHECK();
  if (fallback_rows) {
    MDE_CUDA_TRY(cudaMemcpyAsync(fallback_rows, hdr + kHdrCount, sizeof(int), cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaStreamSynchronize(st));
  }
  return 0;
}

// Arguments shared by every dense exact search: the query rows [lo, hi) of X (a full search is [0, n)).
bool bad_search_args(const void* X, int64_t n, int d, int64_t lo, int64_t hi, int k, int max_k, const void* idx_out,
                     const void* d2_out, const void* ws) {
  return !X || !idx_out || !d2_out || !ws || n < 2 || d < 1 || k < 1 || k > max_k || k > n - 1 || lo < 0 ||
         hi > n || lo >= hi;
}

// 8-bit input wider than d_max: its tile sums could leave int32 (the caller searches X.float() instead)
template <class T>
bool too_wide(int d) {
  if constexpr (kInt8<T>) return d > knn8_max_d<T>();
  else return false;
}

// mde_knn / mde_knn16 / mde_knn8 / the narrow mde_knn_rows: centring and prep, tiles (in S candidate slices), re-rank of the 32
// candidates (merge of the 32 S), certificate and direct search.
template <class T>
int run_narrow(const T* X, int64_t n, int d, int64_t lo, int64_t hi, int k, int32_t* idx_out, float* d2_out, void* ws,
               size_t ws_bytes, void* stream, int* fallback_rows) {
  if (bad_search_args(X, n, d, lo, hi, k, kMaxK, idx_out, d2_out, ws)) return MDE_E_INVALID;
  if (n > (1ll << 31) - kTileN || too_wide<T>(d)) return MDE_E_UNSUPPORTED;
  const KnnLayout L = knn_layout(n, d, hi - lo, kNarrow, kOpKind<T>);
  if (ws_bytes < L.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  EncodeTiledFn enc = nullptr;
  int rc;
  if ((rc = tensor_map_encoder(&enc))) return rc;
  uint8_t* w = static_cast<uint8_t*>(ws);
  OpT<T>* Xh = reinterpret_cast<OpT<T>*>(w + L.off_h);
  __nv_bfloat16* Xl = reinterpret_cast<__nv_bfloat16*>(w + L.off_l);
  AccT<T>* norms = reinterpret_cast<AccT<T>*>(w + L.off_norm);
  int32_t* ci = reinterpret_cast<int32_t*>(w + L.off_ci);
  AccT<T>* cv = reinterpret_cast<AccT<T>*>(w + L.off_cv);
  CUtensorMap mh, ml;
  if ((rc = make_map(enc, &mh, Xh, L.n_pad, L.k_pad, kTileM, Operand<T>::kMapType))) return rc;
  if ((rc = make_map(enc, &ml, Xl, L.n_pad, L.k_pad, kTileM, Operand<T>::kMapType))) return rc;
  if ((rc = centre_and_prep<T>(X, n, d, L, w, st))) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    MDE_CUDA_TRY(cudaFuncSetAttribute(knn_tile_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  const QueryRange qr{lo / kTileN * kTileN, lo, hi, L.slices};
  const dim3 grid((unsigned)((hi - qr.base + kTileM - 1) / kTileM), (unsigned)L.slices);
  knn_tile_kernel<T><<<grid, kThreads, kSmemBytes, st>>>(mh, ml, norms, n, L.n_pad, L.k_pad, qr, ci, cv);
  MDE_LAUNCH_CHECK();
  return rerank_certify<T>(kKK, X, n, d, lo, hi, k, idx_out, d2_out, L, w, st, fallback_rows);
}

// mde_knn_wide (KK = 96, TN = 128) and mde_knn_long (KK = 288, TN = 64), their 16-bit entries and the wide
// mde_knn_rows: centring and prep, tiles (in S candidate slices), re-rank of all KK candidates (merge of the KK S),
// certificate and direct search.
template <class T, int KK, int TN>
int run_wide(const T* X, int64_t n, int d, int64_t lo, int64_t hi, int k, int max_k, int32_t* idx_out, float* d2_out,
             void* ws, size_t ws_bytes, void* stream, int* fallback_rows, bool split = KK != kLongKK) {
  if (bad_search_args(X, n, d, lo, hi, k, max_k, idx_out, d2_out, ws)) return MDE_E_INVALID;
  if (n > (1ll << 31) - kTileN || too_wide<T>(d)) return MDE_E_UNSUPPORTED;
  const KnnLayout L = knn_layout(n, d, hi - lo, Shape{kWideTileM, TN, KK, split}, kOpKind<T>);
  if (ws_bytes < L.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  EncodeTiledFn enc = nullptr;
  int rc;
  if ((rc = tensor_map_encoder(&enc))) return rc;
  uint8_t* w = static_cast<uint8_t*>(ws);
  OpT<T>* Xh = reinterpret_cast<OpT<T>*>(w + L.off_h);
  __nv_bfloat16* Xl = reinterpret_cast<__nv_bfloat16*>(w + L.off_l);
  AccT<T>* norms = reinterpret_cast<AccT<T>*>(w + L.off_norm);
  int32_t* ci = reinterpret_cast<int32_t*>(w + L.off_ci);
  AccT<T>* cv = reinterpret_cast<AccT<T>*>(w + L.off_cv);
  constexpr CUtensorMapDataType kType = Operand<T>::kMapType;
  CUtensorMap mah, mal, mh, ml;  // query operand in 64-row boxes, candidate operand in TN-row boxes
  if ((rc = make_map(enc, &mah, Xh, L.n_pad, L.k_pad, kWideTileM, kType))) return rc;
  if ((rc = make_map(enc, &mal, Xl, L.n_pad, L.k_pad, kWideTileM, kType))) return rc;
  if ((rc = make_map(enc, &mh, Xh, L.n_pad, L.k_pad, TN, kType))) return rc;
  if ((rc = make_map(enc, &ml, Xl, L.n_pad, L.k_pad, TN, kType))) return rc;
  if ((rc = centre_and_prep<T>(X, n, d, L, w, st))) return rc;
  constexpr int kSmem = kWideSmemBytes<KK, TN>;
  static bool attr_set = false;
  if (!attr_set) {
    MDE_CUDA_TRY(cudaFuncSetAttribute(knn_wide_tile_kernel<T, KK, TN>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      kSmem));
    attr_set = true;
  }
  const QueryRange qr{lo / kTileN * kTileN, lo, hi, L.slices};
  const dim3 grid((unsigned)((hi - qr.base + kWideTileM - 1) / kWideTileM), (unsigned)L.slices);
  knn_wide_tile_kernel<T, KK, TN><<<grid, kWideThreads, kSmem, st>>>(mah, mal, mh, ml, norms, n, L.n_pad, L.k_pad, qr,
                                                                     ci, cv);
  MDE_LAUNCH_CHECK();
  return rerank_certify<T>(KK, X, n, d, lo, hi, k, idx_out, d2_out, L, w, st, fallback_rows);
}

// The 16-bit and 8-bit entries: dtype code -> element type, MDE_E_INVALID for an unknown code (before any CUDA call).
template <template <class> class Run, class... A>
int by_dtype(const void* X, int dtype, A... args) {
  if (dtype == MDE_DTYPE_FP16) return Run<__half>::call(static_cast<const __half*>(X), args...);
  if (dtype == MDE_DTYPE_BF16) return Run<__nv_bfloat16>::call(static_cast<const __nv_bfloat16*>(X), args...);
  return MDE_E_INVALID;
}
template <template <class> class Run, class... A>
int by_dtype8(const void* X, int dtype, A... args) {
  if (dtype == MDE_DTYPE_U8) return Run<uint8_t>::call(static_cast<const uint8_t*>(X), args...);
  if (dtype == MDE_DTYPE_S8) return Run<int8_t>::call(static_cast<const int8_t*>(X), args...);
  return MDE_E_INVALID;
}
template <class T>
struct Narrow {
  static int call(const T* X, int64_t n, int d, int k, int32_t* i, float* d2, void* ws, size_t b, void* st, int* fb) {
    return run_narrow<T>(X, n, d, 0, n, k, i, d2, ws, b, st, fb);
  }
};
template <class T>
struct Wide {
  static int call(const T* X, int64_t n, int d, int k, int32_t* i, float* d2, void* ws, size_t b, void* st, int* fb) {
    return run_wide<T, kWideKK, kTileN>(X, n, d, 0, n, k, kWideMaxK, i, d2, ws, b, st, fb);
  }
};
template <class T>
struct Long {
  static int call(const T* X, int64_t n, int d, int k, int32_t* i, float* d2, void* ws, size_t b, void* st, int* fb) {
    return run_wide<T, kLongKK, kLongTileN>(X, n, d, 0, n, k, kLongMaxK, i, d2, ws, b, st, fb);
  }
};
// mde_knn_long_rows / mde_knn16_long_rows / mde_knn8_long_rows: the long search, split into candidate slices
template <class T>
struct LongRows {
  static int call(const T* X, int64_t n, int d, int64_t lo, int64_t hi, int k, int32_t* i, float* d2, void* ws,
                  size_t b, void* st, int* fb) {
    return run_wide<T, kLongKK, kLongTileN>(X, n, d, lo, hi, k, kLongMaxK, i, d2, ws, b, st, fb, true);
  }
};
// mde_knn_rows / mde_knn16_rows / mde_knn8_rows: the narrow search for k <= 24, the wide one up to 64
template <class T>
struct Rows {
  static int call(const T* X, int64_t n, int d, int64_t lo, int64_t hi, int k, int32_t* i, float* d2, void* ws,
                  size_t b, void* st, int* fb) {
    if (k > kMaxK) return run_wide<T, kWideKK, kTileN>(X, n, d, lo, hi, k, kWideMaxK, i, d2, ws, b, st, fb);
    return run_narrow<T>(X, n, d, lo, hi, k, i, d2, ws, b, st, fb);
  }
};

int layout_bytes(int64_t n, int d, Shape sh, OpKind op, size_t* bytes) {
  if (!bytes || n < 2 || d < 1) return MDE_E_INVALID;
  *bytes = knn_layout(n, d, n, sh, op).total;
  return 0;
}

int rows_layout_bytes(int64_t n, int d, int64_t rows, int k, OpKind op, size_t* bytes) {
  if (!bytes || n < 2 || d < 1 || rows < 1 || rows > n || k < 1 || k > kWideMaxK || k > n - 1) return MDE_E_INVALID;
  *bytes = knn_layout(n, d, rows, k > kMaxK ? kWide : kNarrow, op).total;
  return 0;
}

int long_rows_layout_bytes(int64_t n, int d, int64_t rows, int k, OpKind op, size_t* bytes) {
  if (!bytes || n < 2 || d < 1 || rows < 1 || rows > n || k < 1 || k > kLongMaxK || k > n - 1) return MDE_E_INVALID;
  *bytes = knn_layout(n, d, rows, kLongRows, op).total;
  return 0;
}

}  // namespace

extern "C" {

int mde_knn_max_k(void) { return kMaxK; }

int mde_knn_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kNarrow, kOpSplit, bytes); }

int mde_knn_ex(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
               void* stream, int* fallback_rows) {
  return run_narrow<float>(X, n, d, 0, n, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
            void* stream) {
  return mde_knn_ex(X, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_wide_max_k(void) { return kWideMaxK; }

int mde_knn_wide_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kWide, kOpSplit, bytes); }

int mde_knn_wide_ex(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                    size_t ws_bytes, void* stream, int* fallback_rows) {
  return run_wide<float, kWideKK, kTileN>(X, n, d, 0, n, k, kWideMaxK, idx_out, d2_out, ws, ws_bytes, stream,
                                          fallback_rows);
}

int mde_knn_wide(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                 size_t ws_bytes, void* stream) {
  return mde_knn_wide_ex(X, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_long_max_k(void) { return kLongMaxK; }

int mde_knn_long_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kLong, kOpSplit, bytes); }

int mde_knn_long_ex(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                    size_t ws_bytes, void* stream, int* fallback_rows) {
  return run_wide<float, kLongKK, kLongTileN>(X, n, d, 0, n, k, kLongMaxK, idx_out, d2_out, ws, ws_bytes, stream,
                                              fallback_rows);
}

int mde_knn_long(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                 size_t ws_bytes, void* stream) {
  return mde_knn_long_ex(X, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_rows_ws_bytes(int64_t n, int d, int64_t rows, int k, size_t* bytes) {
  return rows_layout_bytes(n, d, rows, k, kOpSplit, bytes);
}

int mde_knn_rows(const float* X, int64_t n, int d, int64_t row_begin, int64_t row_end, int k, int32_t* idx_out,
                 float* d2_out, void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return Rows<float>::call(X, n, d, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn_long_rows_ws_bytes(int64_t n, int d, int64_t rows, int k, size_t* bytes) {
  return long_rows_layout_bytes(n, d, rows, k, kOpSplit, bytes);
}

int mde_knn_long_rows(const float* X, int64_t n, int d, int64_t row_begin, int64_t row_end, int k, int32_t* idx_out,
                      float* d2_out, void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return LongRows<float>::call(X, n, d, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn16_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kNarrow, kOp16, bytes); }

int mde_knn16_ex(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                 size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype<Narrow>(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn16(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
              size_t ws_bytes, void* stream) {
  return mde_knn16_ex(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn16_wide_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kWide, kOp16, bytes); }

int mde_knn16_wide_ex(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                      size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype<Wide>(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn16_wide(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                   size_t ws_bytes, void* stream) {
  return mde_knn16_wide_ex(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn16_long_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kLong, kOp16, bytes); }

int mde_knn16_long_ex(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                      size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype<Long>(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn16_long(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                   size_t ws_bytes, void* stream) {
  return mde_knn16_long_ex(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn16_rows_ws_bytes(int64_t n, int d, int64_t rows, int k, size_t* bytes) {
  return rows_layout_bytes(n, d, rows, k, kOp16, bytes);
}

int mde_knn16_rows(const void* X, int dtype, int64_t n, int d, int64_t row_begin, int64_t row_end, int k,
                   int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype<Rows>(X, dtype, n, d, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn16_long_rows_ws_bytes(int64_t n, int d, int64_t rows, int k, size_t* bytes) {
  return long_rows_layout_bytes(n, d, rows, k, kOp16, bytes);
}

int mde_knn16_long_rows(const void* X, int dtype, int64_t n, int d, int64_t row_begin, int64_t row_end, int k,
                        int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype<LongRows>(X, dtype, n, d, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes, stream,
                            fallback_rows);
}

int mde_knn8_max_d(int dtype) {
  if (dtype == MDE_DTYPE_U8) return knn8_max_d<uint8_t>();
  if (dtype == MDE_DTYPE_S8) return knn8_max_d<int8_t>();
  return MDE_E_INVALID;
}

int mde_knn8_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kNarrow, kOp8, bytes); }

int mde_knn8_ex(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype8<Narrow>(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn8(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
             size_t ws_bytes, void* stream) {
  return mde_knn8_ex(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn8_wide_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kWide, kOp8, bytes); }

int mde_knn8_wide_ex(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                     size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype8<Wide>(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn8_wide(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                  size_t ws_bytes, void* stream) {
  return mde_knn8_wide_ex(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn8_long_ws_bytes(int64_t n, int d, size_t* bytes) { return layout_bytes(n, d, kLong, kOp8, bytes); }

int mde_knn8_long_ex(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                     size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype8<Long>(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn8_long(const void* X, int dtype, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                  size_t ws_bytes, void* stream) {
  return mde_knn8_long_ex(X, dtype, n, d, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn8_rows_ws_bytes(int64_t n, int d, int64_t rows, int k, size_t* bytes) {
  return rows_layout_bytes(n, d, rows, k, kOp8, bytes);
}

int mde_knn8_rows(const void* X, int dtype, int64_t n, int d, int64_t row_begin, int64_t row_end, int k,
                  int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype8<Rows>(X, dtype, n, d, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes, stream, fallback_rows);
}

int mde_knn8_long_rows_ws_bytes(int64_t n, int d, int64_t rows, int k, size_t* bytes) {
  return long_rows_layout_bytes(n, d, rows, k, kOp8, bytes);
}

int mde_knn8_long_rows(const void* X, int dtype, int64_t n, int d, int64_t row_begin, int64_t row_end, int k,
                       int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return by_dtype8<LongRows>(X, dtype, n, d, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes, stream,
                             fallback_rows);
}

// host-side debug entry point: the certificate's gamma for 8-bit input of d columns (cert_bound); -1 for d < 1
double mde_dbg_knn8_gamma(int d) { return d < 1 ? -1.0 : knn8_gamma(d); }

// host-side debug entry point: the candidate slices (mde_logic.h: knn_slices) of a search of `rows` query rows
// against n rows with k neighbours (the narrow search up to k = 24, the wide one up to 64); -1 for bad arguments
int mde_dbg_knn_slices(int64_t n, int64_t rows, int k) {
  if (n < 2 || rows < 1 || rows > n || k < 1 || k > kWideMaxK) return -1;
  return search_slices(n, rows, k > kMaxK ? kWide : kNarrow);
}

// host-side debug entry point: the candidate slices of the long row search (mde_knn_long_rows) of `rows` query rows
// against n rows, 1 <= k <= 256: knn_slices with TM = TN = 64; -1 for bad arguments
int mde_dbg_knn_long_slices(int64_t n, int64_t rows, int k) {
  if (n < 2 || rows < 1 || rows > n || k < 1 || k > kLongMaxK) return -1;
  return search_slices(n, rows, kLongRows);
}

}  // extern "C"
