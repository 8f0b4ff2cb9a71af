// mde_knn_sparse.cu -- exact k-nearest neighbours and pair distances of the rows of a CSR data matrix (SURVEY
// section 8 row f3, sparse input).
//
// The reference hands a scipy.sparse matrix to pynndescent for the k-NN and to scipy for the distances of sampled
// pairs (pymde/preprocess/data_matrix.py:59-70).  Densifying costs n d 4 bytes, which a TF-IDF or count matrix
// cannot afford, so this file works from the CSR arrays alone (int64 indptr, int32 indices strictly increasing within
// a row, fp32 values):
//
//   prep     validate the CSR, ||x||^2 (fp64 sums, fp32; +inf on padding rows) and a column histogram; a permutation
//            of the features by descending document frequency (CUB radix sort); every row re-sorted under it (one
//            radix sort on the key (row, new column)); one occupancy bitmap per 128-row tile with one bit per
//            64-feature K block.  Frequent features land in the first K blocks, so most tiles touch few of the rest.
//   tiles    one CTA per 128 query rows sweeps every candidate tile, as knn_tile_kernel in mde_knn.cu does.  For a
//            (query tile, candidate tile) pair only the K blocks set in both bitmaps are visited; a pair with none has
//            cross terms of exactly 0.  All 256 threads build each 128 x 64 operand block (bf16 hi and lo of both
//            tiles) straight from CSR: a thread owns one row, zeroes its 128-byte swizzled rows with 16-byte stores
//            and scatters the row's entries of the block, its cursor advancing monotonically through the visited
//            blocks.  fence.proxy.async makes these generic-proxy writes visible to wgmma (async proxy); block j's
//            scatter into one stage overlaps the wgmmas of block j - 1 on the other.  Two consumer warpgroups issue
//            wgmma.m64n128k16 with Ah Bh^T + Ah Bl^T + Al Bh^T and keep a running top-32 per row, ordered by
//            (approximate distance, index).
//   re-rank  sum (q - x)^2 over each candidate by a sorted merge of the two rows, in fp64, rounded once to fp32; the
//            k smallest by (distance, index).  The result is fully determined, ties included.
//
// mde_knn_csr_wide (24 < k <= 64): the same preparation; knn_csr_wide_tile_kernel sweeps 64 query rows per CTA and
// keeps KK = 96 candidates per row in shared memory (mde_knn_select.cuh); the re-rank merges all 96.
// mde_knn_csr_long (k <= 256): the same kernel with KK = 288 on candidate tiles of 64 rows (one warpgroup); the
// re-rank merges all 288.
//
// mde_knn_csr_rows searches a range of query rows against all n rows with the narrow, wide or long tiles (every full
// search is the range [0, n) in one slice).  The preparation still covers the whole matrix; the tiles sweep only the
// query tiles, aligned as in the full search.  When those leave SMs idle the narrow and wide sweeps are split into S
// candidate slices (blockIdx.y; S from mde_logic.h::knn_slices), and knn_csr_merge_kernel keeps the KK smallest of a
// row's S lists by the tiles' own (score, index) order -- the full search's candidates -- for the re-rank
// (DESIGN 11.8).
//
// mde_pair_dist_csr: ||a - b|| of given pairs by the same sorted merge, fp64, sqrt in fp64, one rounding.
#include <cub/cub.cuh>
#include <cuda_bf16.h>

#include <climits>
#include <cstdint>

#include "mde_common.cuh"
#include "mde_knn_csr.cuh"
#include "mde_knn_select.cuh"
#include "mde_logic.h"
#include "mde_tma.cuh"
#include "mde_wgmma.cuh"

using namespace mde;

namespace {

constexpr int kTileM = 128;                 // query rows per CTA (two warpgroups of 64)
constexpr int kTileN = 128;                 // candidates per tile = wgmma N
constexpr int kBlockK = 64;                 // bf16 elements per 128-byte swizzle row
constexpr int kWgmmaK = 16;
constexpr int kStages = 2;
constexpr int kKK = 32;                     // candidates kept per row before the exact re-rank
constexpr int kMaxK = 24;
constexpr int kRowBytes = kBlockK * 2;      // 128
constexpr int kOpBytes = 128 * kRowBytes;   // 16 KB: one 128-row operand block (hi or lo)
constexpr int kStageBytes = 4 * kOpBytes;   // A hi, A lo, B hi, B lo = 64 KB
constexpr int kThreads = 256;               // two warpgroups: each thread builds one operand row, each warpgroup
                                            // consumes 64 query rows
constexpr int kChunkWords = 128;            // bitmap words intersected per pass (4096 K blocks)
constexpr int kAccStride = kTileN + 2;
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /* alignment slack */ + kTileM * kAccStride * 4 +
                           kTileN * 4 /* norms */ + kChunkWords * 32 * 4 /* visited-block list */;
static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

// wide (k <= 64) and long (k <= 256) searches: 64 query rows per CTA, running top-KK lists in shared memory,
// candidate tiles of TN = 128 (wide) or 64 (long) rows, one warpgroup per 64 candidates of a tile
constexpr int kWideTileM = 64;
constexpr int kAOpBytes = kWideTileM * kRowBytes;              // 8 KB: one 64-row query operand block (hi or lo)
constexpr int kLongTileN = 64;

template <int TN>
constexpr int kWideStageBytes = 2 * kAOpBytes + 2 * TN * kRowBytes;  // A hi, A lo, B hi, B lo
// The staged accumulators [64][TN + 2] share the stage buffers: the tile's last wgmmas are done before they are
// written, and the next tile's first operand block is built after the scan.
template <int KK, int TN>
constexpr int kWideSmemBytes = kStages * kWideStageBytes<TN> + 1024 /* alignment slack */ + TN * 4 /* norms */ +
                               kChunkWords * 32 * 4 /* visited-block list */ +
                               kWideTileM * WideList<KK>::kStride * 8 /* lists */;
// long: the 148.5 KB of lists leave 2 x 32 KB stages of 64-wide candidate tiles (CUB's scan storage is static)
static_assert(kWideSmemBytes<kWideKK, kTileN> <= 227 * 1024, "H100: at most 227 KB of shared memory per block");
static_assert(kWideSmemBytes<kLongKK, kLongTileN> + 768 /* CUB scan, 672 B */ <= 227 * 1024,
              "H100: at most 227 KB of shared memory per block, static storage included");

constexpr float kInf = __builtin_huge_valf();

__device__ __forceinline__ bool before(float d1, int i1, float d2, int i2) { return d1 < d2 || (d1 == d2 && i1 < i2); }

// Replace the worst of the KK kept candidates by (dist, col); the new worst is the largest (distance, index).
__device__ __forceinline__ void keep_candidate(float (&bd)[kKK], int (&bi)[kKK], float dist, int col, float& thr,
                                               int& thi, int& worst) {
#pragma unroll
  for (int q = 0; q < kKK; ++q) {
    if (q == worst) { bd[q] = dist; bi[q] = col; }
  }
  float m = bd[0]; int mi = bi[0], w = 0;
#pragma unroll
  for (int q = 1; q < kKK; ++q) {
    if (before(m, mi, bd[q], bi[q])) { m = bd[q]; mi = bi[q]; w = q; }
  }
  thr = m; thi = mi; worst = w;
}

// ---------------------------------------------------------------------------------------------------------------
// prep
// ---------------------------------------------------------------------------------------------------------------
// One warp per row: checks the row's CSR (bounds, indices in [0, d), strictly increasing) and sets *bad otherwise;
// optionally counts each column and writes the fp32-rounded fp64 squared norm.  Padding rows get +inf norms.
__global__ void __launch_bounds__(256)
csr_check_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                 const float* __restrict__ values, int64_t n, int d, int64_t nnz, int64_t n_pad,
                 int* __restrict__ bad, int32_t* __restrict__ col_count, float* __restrict__ norms) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) {
    if (norms && row < n_pad && lane == 0) norms[row] = kInf;
    return;
  }
  const int64_t b = indptr[row], e = indptr[row + 1];
  if (b < 0 || e < b || e > nnz || (row == 0 && b != 0) || (row == n - 1 && e != nnz)) {
    if (lane == 0) atomicOr(bad, 1);
    return;
  }
  double acc = 0.0;
  bool ok = true;
  for (int64_t p = b + lane; p < e; p += 32) {
    const int c = indices[p];
    if (c < 0 || c >= d || (p > b && indices[p - 1] >= c)) { ok = false; continue; }
    if (col_count) atomicAdd(col_count + c, 1);
    const double x = values[p];
    acc += x * x;
  }
  if (!__all_sync(kFull, ok) && lane == 0) atomicOr(bad, 1);
  if (norms) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (lane == 0) norms[row] = (float)acc;
  }
}

__global__ void iota_kernel(int32_t* __restrict__ v, int d) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < d) v[i] = i;
}

__global__ void invert_perm_kernel(const int32_t* __restrict__ col_sorted, int d, int32_t* __restrict__ perm) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < d) perm[col_sorted[i]] = i;
}

// One warp per row: sort keys (row << col_bits | new column) and the tile occupancy bitmaps.
__global__ void __launch_bounds__(256)
csr_keys_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                const int32_t* __restrict__ perm, int64_t n, int col_bits, int nwords, uint64_t* __restrict__ keys,
                uint32_t* __restrict__ bitmap) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  uint32_t* bm = bitmap + (row / kTileM) * nwords;
  const int64_t e = indptr[row + 1];
  for (int64_t p = indptr[row] + lane; p < e; p += 32) {
    const int c = perm[indices[p]];
    keys[p] = ((uint64_t)row << col_bits) | (uint32_t)c;
    const int kb = c / kBlockK;
    atomicOr(bm + (kb >> 5), 1u << (kb & 31));
  }
}

__global__ void key_to_col_kernel(const uint64_t* __restrict__ keys, int64_t nnz, uint64_t mask,
                                  int32_t* __restrict__ cols) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nnz) cols[i] = (int32_t)(keys[i] & mask);
}

// ---------------------------------------------------------------------------------------------------------------
// tiles
// ---------------------------------------------------------------------------------------------------------------
// CTA (x, y) sweeps query tile qr.base / 128 + x against candidate slice y (QueryRange); query rows outside
// [qr.lo, qr.hi) write nothing.
__global__ void __launch_bounds__(kThreads, 1)
knn_csr_tile_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                    const float* __restrict__ vals, const float* __restrict__ norms,
                    const uint32_t* __restrict__ bitmap, int nwords, int64_t n, int num_tiles, QueryRange qr,
                    int32_t* __restrict__ cand_idx, float* __restrict__ cand_val) {
  extern __shared__ uint8_t smem_raw[];
  // carve: [stages x 64 KB, 1024-aligned] | staged accumulators [128][kAccStride] | norms[128] | visited blocks
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  float* s_acc = reinterpret_cast<float*>(gen + kStages * kStageBytes);
  float* s_norm = s_acc + kTileM * kAccStride;
  int* s_list = reinterpret_cast<int*>(s_norm + kTileN);
  using Scan = cub::BlockScan<int, kThreads>;
  __shared__ typename Scan::TempStorage scan_tmp;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t row0 = qr.base + (int64_t)blockIdx.x * kTileM;
  const uint32_t* abm = bitmap + (row0 / kTileM) * nwords;
  const int t_begin = qr.slice_begin(num_tiles), t_end = qr.slice_begin(num_tiles, 1);

  // ----- builder role: thread tid owns operand row tid & 127 of A (query tile, tid < 128) or B (candidate tile)
  const bool is_b = tid >= 128;
  const int orow = tid & 127;
  const uint32_t my_off = (is_b ? 2 * kOpBytes : 0) + orow * kRowBytes;
  const int swz = orow & 7;
  int64_t a_beg = 0, a_end = 0;
  if (!is_b && row0 + orow < n) { a_beg = indptr[row0 + orow]; a_end = indptr[row0 + orow + 1]; }

  // ----- consumer role: warpgroup wg owns query rows row0 + 64 wg .. + 63
  const int wg = warp >> 2;
  const int et = tid & 127;
  float* acc_s = s_acc + wg * 64 * kAccStride;
  const int lrow = et >> 1, half = et & 1;
  const int64_t row = row0 + wg * 64 + lrow;
  const int frow = 16 * (warp & 3) + (lane >> 2), fcol = 2 * (lane & 3);

  float bd[kKK];
  int bi[kKK];
#pragma unroll
  for (int q = 0; q < kKK; ++q) { bd[q] = kInf; bi[q] = INT_MAX; }
  float thr = kInf;
  int thi = INT_MAX, worst = 0;
  float acc[64];

  int stage = 0;
  for (int t = t_begin; t < t_end; ++t) {
    int64_t p = a_beg, end = a_end;
    if (is_b) {
      const int64_t r = (int64_t)t * kTileN + orow;
      p = end = 0;
      if (r < n) { p = indptr[r]; end = indptr[r + 1]; }
    }
    int cur = p < end ? cols[p] : INT_MAX;
    const uint32_t* bbm = bitmap + (int64_t)t * nwords;
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.0f;

    for (int w0 = 0; w0 < nwords; w0 += kChunkWords) {
      __syncthreads();  // every thread is done with s_list (and, on the first chunk, with the last tile's scan)
      uint32_t m = 0;
      if (tid < kChunkWords && w0 + tid < nwords) m = __ldg(abm + w0 + tid) & __ldg(bbm + w0 + tid);
      int pos, total;
      Scan(scan_tmp).ExclusiveSum(__popc(m), pos, total);
      for (; m; m &= m - 1) s_list[pos++] = (w0 + tid) * 32 + (__ffs(m) - 1);
      __syncthreads();
      for (int i = 0; i < total; ++i) {
        const int lo = s_list[i] * kBlockK, hi = lo + kBlockK;
        // the stage was last read by the wgmmas of block i - 2, which every warpgroup waited for before the
        // barrier of block i - 1
        uint8_t* rh = gen + stage * kStageBytes + my_off;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          reinterpret_cast<uint4*>(rh)[c] = make_uint4(0, 0, 0, 0);
          reinterpret_cast<uint4*>(rh + kOpBytes)[c] = make_uint4(0, 0, 0, 0);
        }
        while (cur < hi) {
          if (cur >= lo) {
            const float x = vals[p];
            const __nv_bfloat16 h = __float2bfloat16_rn(x);
            const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
            const int k = cur - lo;
            const int off = (((k >> 3) ^ swz) << 4) | ((k & 7) << 1);
            *reinterpret_cast<__nv_bfloat16*>(rh + off) = h;
            *reinterpret_cast<__nv_bfloat16*>(rh + kOpBytes + off) = l;
          }
          ++p;
          cur = p < end ? cols[p] : INT_MAX;
        }
        fence_proxy_async();  // generic-proxy stores above, read next by wgmma (async proxy)
        wgmma_wait_all();     // this warpgroup's wgmmas of block i - 1 are done with the other stage
        __syncthreads();
        const uint32_t sa = base + stage * kStageBytes;
        const uint64_t ah = smem_desc_sw128(sa + wg * 64 * kRowBytes);
        const uint64_t al = smem_desc_sw128(sa + kOpBytes + wg * 64 * kRowBytes);
        const uint64_t bh = smem_desc_sw128(sa + 2 * kOpBytes), bl = smem_desc_sw128(sa + 3 * kOpBytes);
#pragma unroll
        for (int q = 0; q < 64; ++q) fence_operand(acc[q]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
          const uint64_t adv = (uint64_t)((k * kWgmmaK * 2) >> 4);
          wgmma_bf16(acc, ah + adv, bh + adv, 1u);
          wgmma_bf16(acc, ah + adv, bl + adv, 1u);
          wgmma_bf16(acc, al + adv, bh + adv, 1u);
        }
        wgmma_commit();
        stage ^= 1;
      }
    }
    wgmma_wait_all();
#pragma unroll
    for (int q = 0; q < 64; ++q) fence_operand(acc[q]);
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      *reinterpret_cast<float2*>(acc_s + frow * kAccStride + 8 * j + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(acc_s + (frow + 8) * kAccStride + 8 * j + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    if (tid < kTileN) s_norm[tid] = __ldg(norms + (int64_t)t * kTileN + tid);
    __syncthreads();
    const float* arow = acc_s + lrow * kAccStride;
#pragma unroll 4
    for (int i = 0; i < kTileN / 2; ++i) {
      const int c = 2 * i + half;
      const float dist = fmaf(-2.0f, arow[c], s_norm[c]);
      const int col = t * kTileN + c;
      if (before(dist, col, thr, thi) && col != row && col < n) keep_candidate(bd, bi, dist, col, thr, thi, worst);
    }
  }
  // merge the two half-row lists: the odd-column thread hands its list to the even-column thread
  __syncthreads();
  float* xd = acc_s + lrow * kAccStride;
  int* xi = reinterpret_cast<int*>(xd + kKK);
  if (half) {
#pragma unroll
    for (int q = 0; q < kKK; ++q) { xd[q] = bd[q]; xi[q] = bi[q]; }
  }
  __syncthreads();
  if (!half) {
    for (int q = 0; q < kKK; ++q) {
      if (before(xd[q], xi[q], thr, thi)) keep_candidate(bd, bi, xd[q], xi[q], thr, thi, worst);
    }
    if (qr.has(row)) {
      const int64_t o = qr.list(row) * kKK;
#pragma unroll
      for (int q = 0; q < kKK; ++q) {
        cand_idx[o + q] = bi[q] == INT_MAX ? -1 : bi[q];
        cand_val[o + q] = bd[q];
      }
    }
  }
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------
// re-rank: merge_dist2 (mde_knn_csr.cuh) of a row's candidates, the k smallest in ascending order
// (namespace mde, declared in mde_knn_csr.cuh: mde_knn_approx.cu re-ranks its lists with the same kernels)
// ---------------------------------------------------------------------------------------------------------------
namespace mde {

// One warp per row r of rows (query row lo + r), lane q re-ranks candidate q; the k smallest (distance, index) in
// ascending order.
__global__ void __launch_bounds__(256)
knn_csr_rerank_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                      const float* __restrict__ vals, int64_t lo, int64_t rows, const int32_t* __restrict__ cand_idx,
                      int k, int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int c = cand_idx[row * kKK + lane];
  const float my_d = c >= 0 ? (float)merge_dist2(indptr, cols, vals, lo + row, c) : kInf;
  const int mine = c >= 0 ? c : INT_MAX;  // missing candidates last
  int rank = 0;
  for (int q = 0; q < kKK; ++q) {
    const float od = __shfl_sync(kFull, my_d, q);
    const int oi = __shfl_sync(kFull, mine, q);
    if (before(od, oi, my_d, mine)) ++rank;
  }
  if (rank < k) {
    out_idx[row * k + rank] = mine;
    out_d2[row * k + rank] = my_d;
  }
}

}  // namespace mde

namespace {

// ---------------------------------------------------------------------------------------------------------------
// wide tiles (k <= 64, KK = 96, TN = 128) and long tiles (k <= 256, KK = 288, TN = 64): as knn_csr_tile_kernel for
// 64 query rows, one running top-KK per row in shared memory; warpgroup wg issues wgmma.m64n64k16 on candidates
// 64 wg .. 64 wg + 63 of the tile.  CTA (x, y) sweeps the 64 query rows qr.base + 64 x .. against candidate slice y
// (QueryRange); query rows outside [qr.lo, qr.hi) write nothing.
// ---------------------------------------------------------------------------------------------------------------
template <int KK, int TN>
__global__ void __launch_bounds__(2 * TN, 1)
knn_csr_wide_tile_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                         const float* __restrict__ vals, const float* __restrict__ norms,
                         const uint32_t* __restrict__ bitmap, int nwords, int64_t n, int num_tiles, QueryRange qr,
                         int32_t* __restrict__ cand_idx, float* __restrict__ cand_val) {
  static_assert(TN == 64 || TN == 128, "one or two warpgroups");
  constexpr int kThreadsT = 2 * TN;                  // one warpgroup per 64 candidates of a tile
  constexpr int kBuilders = kWideTileM + TN;         // one builder thread per operand row
  constexpr int kBOpBytes = TN * kRowBytes;
  constexpr int kStageB = kWideStageBytes<TN>;
  constexpr int kAccS = TN + 2;
  constexpr int kStride = WideList<KK>::kStride;
  static_assert(kWideTileM * kAccS * 4 <= kStages * kStageB, "the staged accumulators fit in the stage buffers");
  static_assert(kChunkWords <= kThreadsT, "one bitmap word per thread");
  extern __shared__ uint8_t smem_raw[];
  // carve: [stages x kStageB, 1024-aligned; staged accumulators [64][kAccS] at its start between tiles] | norms[TN] |
  //        visited blocks | list distances [64][kStride] | list indices [64][kStride]
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  float* s_acc = reinterpret_cast<float*>(gen);
  float* s_norm = reinterpret_cast<float*>(gen + kStages * kStageB);
  int* s_list = reinterpret_cast<int*>(s_norm + TN);
  float* s_ld = reinterpret_cast<float*>(s_list + kChunkWords * 32);
  int* s_li = reinterpret_cast<int*>(s_ld + kWideTileM * kStride);
  using Scan = cub::BlockScan<int, kThreadsT>;
  __shared__ typename Scan::TempStorage scan_tmp;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t row0 = qr.base + (int64_t)blockIdx.x * kWideTileM;
  // the query rows use the bitmap of their 128-row tile, and so do the candidate rows: a superset of their own
  // blocks (a block only other rows of that tile occupy is built with zero rows and adds exactly 0)
  const uint32_t* abm = bitmap + (row0 / kTileM) * nwords;
  const int t_begin = qr.slice_begin(num_tiles), t_end = qr.slice_begin(num_tiles, 1);

  // ----- builder role: thread tid owns operand row tid of A (query rows, tid < 64) or row tid - 64 of B (up to
  // tid 64 + TN - 1); with TN = 128, warps 6 and 7 build nothing
  const bool builder = tid < kBuilders;  // (warp-uniform)
  const bool is_b = tid >= kWideTileM;
  const int orow = is_b ? tid - kWideTileM : tid;
  const uint32_t my_off = (is_b ? 2 * kAOpBytes : 0) + orow * kRowBytes;
  const uint32_t lo_off = is_b ? kBOpBytes : kAOpBytes;  // from the hi block to the lo block of the operand
  const int swz = orow & 7;
  int64_t a_beg = 0, a_end = 0;
  if (!is_b && row0 + orow < n) { a_beg = indptr[row0 + orow]; a_end = indptr[row0 + orow + 1]; }

  // ----- consumer role: warpgroup wg multiplies the 64 query rows by candidates 64 wg .. 64 wg + 63 of the tile;
  // the scanners, threads 0-127, own the query rows, two adjacent lanes per row
  const int wg = warp >> 2;
  const bool scanner = tid < 128;  // (warp-uniform)
  const int lrow = (tid & 127) >> 1, half = tid & 1;
  const int64_t row = row0 + lrow;
  const int frow = 16 * (warp & 3) + (lane >> 2), fcol = 64 * wg + 2 * (lane & 3);
  WideList<KK> list;
  if (scanner) list.init(s_ld + lrow * kStride, s_li + lrow * kStride, half);
  float acc[32];

  int stage = 0;
  for (int t = t_begin; t < t_end; ++t) {
    int64_t p = a_beg, end = a_end;
    if (is_b) {
      const int64_t r = (int64_t)t * TN + orow;
      p = end = 0;
      if (builder && r < n) { p = indptr[r]; end = indptr[r + 1]; }
    }
    int cur = p < end ? cols[p] : INT_MAX;
    const uint32_t* bbm = bitmap + ((int64_t)t * TN / kTileM) * nwords;
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.0f;

    for (int w0 = 0; w0 < nwords; w0 += kChunkWords) {
      __syncthreads();  // every thread is done with s_list (and, on the first chunk, with the last tile's scan)
      uint32_t m = 0;
      if (tid < kChunkWords && w0 + tid < nwords) m = __ldg(abm + w0 + tid) & __ldg(bbm + w0 + tid);
      int pos, total;
      Scan(scan_tmp).ExclusiveSum(__popc(m), pos, total);
      for (; m; m &= m - 1) s_list[pos++] = (w0 + tid) * 32 + (__ffs(m) - 1);
      __syncthreads();
      for (int i = 0; i < total; ++i) {
        const int lo = s_list[i] * kBlockK, hi = lo + kBlockK;
        // the stage was last read by the wgmmas of block i - 2, which the consumers waited for before the barrier
        // of block i - 1
        uint8_t* rh = gen + stage * kStageB + my_off;
        if (builder) {
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            reinterpret_cast<uint4*>(rh)[c] = make_uint4(0, 0, 0, 0);
            reinterpret_cast<uint4*>(rh + lo_off)[c] = make_uint4(0, 0, 0, 0);
          }
        }
        while (cur < hi) {
          if (cur >= lo) {
            const float x = vals[p];
            const __nv_bfloat16 h = __float2bfloat16_rn(x);
            const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
            const int k = cur - lo;
            const int off = (((k >> 3) ^ swz) << 4) | ((k & 7) << 1);
            *reinterpret_cast<__nv_bfloat16*>(rh + off) = h;
            *reinterpret_cast<__nv_bfloat16*>(rh + lo_off + off) = l;
          }
          ++p;
          cur = p < end ? cols[p] : INT_MAX;
        }
        fence_proxy_async();  // generic-proxy stores above, read next by wgmma (async proxy)
        wgmma_wait_all();     // this warpgroup's wgmmas of block i - 1 are done with the other stage
        __syncthreads();
        const uint32_t sa = base + stage * kStageB;
        const uint64_t ah = smem_desc_sw128(sa), al = smem_desc_sw128(sa + kAOpBytes);
        const uint64_t bh = smem_desc_sw128(sa + 2 * kAOpBytes + wg * 64 * kRowBytes);
        const uint64_t bl = smem_desc_sw128(sa + 2 * kAOpBytes + kBOpBytes + wg * 64 * kRowBytes);
#pragma unroll
        for (int q = 0; q < 32; ++q) fence_operand(acc[q]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
          const uint64_t adv = (uint64_t)((k * kWgmmaK * 2) >> 4);
          wgmma_bf16_n64(acc, ah + adv, bh + adv, 1u);
          wgmma_bf16_n64(acc, ah + adv, bl + adv, 1u);
          wgmma_bf16_n64(acc, al + adv, bh + adv, 1u);
        }
        wgmma_commit();
        stage ^= 1;
      }
    }
    wgmma_wait_all();
#pragma unroll
    for (int q = 0; q < 32; ++q) fence_operand(acc[q]);
    __syncthreads();  // every warpgroup's wgmmas are done with the stage buffers that take the accumulators
#pragma unroll
    for (int j = 0; j < 64 / 8; ++j) {
      *reinterpret_cast<float2*>(s_acc + frow * kAccS + 8 * j + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(s_acc + (frow + 8) * kAccS + 8 * j + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    if (tid < TN) s_norm[tid] = __ldg(norms + (int64_t)t * TN + tid);
    __syncthreads();
    if (scanner) {
      // both lanes of the row offer every column, in column order
      const float2* arow = reinterpret_cast<const float2*>(s_acc + lrow * kAccS);
      const float2* sn = reinterpret_cast<const float2*>(s_norm);
#pragma unroll 2
      for (int i = 0; i < TN / 2; ++i) {
        const float2 a = arow[i], s = sn[i];
        const int col = t * TN + 2 * i;
        if (col != row && col < n) list.offer(fmaf(-2.0f, a.x, s.x), col);
        if (col + 1 != row && col + 1 < n) list.offer(fmaf(-2.0f, a.y, s.y), col + 1);
      }
    }
  }
  if (scanner && qr.has(row)) list.store(cand_idx + qr.list(row) * KK, cand_val + qr.list(row) * KK);
}

}  // namespace

namespace mde {

// One warp per row r of rows (query row lo + r), lane q re-ranks candidates q, q + 32, q + 64, ... by the merge of
// knn_csr_rerank_kernel; the k smallest (distance, index) of the KK in ascending order.
template <int KK>
__device__ __forceinline__ void csr_wide_rerank_row(const int64_t* __restrict__ indptr,
                                                    const int32_t* __restrict__ cols, const float* __restrict__ vals,
                                                    int64_t lo, int64_t rows, const int32_t* __restrict__ cand_idx,
                                                    int k, int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  constexpr int kPer = KK / 32;
  float my_d[kPer];
  int mine[kPer];
#pragma unroll
  for (int s = 0; s < kPer; ++s) {
    const int c = cand_idx[row * KK + 32 * s + lane];
    my_d[s] = c >= 0 ? (float)merge_dist2(indptr, cols, vals, lo + row, c) : kInf;
    mine[s] = c >= 0 ? c : INT_MAX;  // missing candidates last
  }
  int rank[kPer] = {};
#pragma unroll
  for (int s2 = 0; s2 < kPer; ++s2) {
    for (int q = 0; q < 32; ++q) {
      const float od = __shfl_sync(kFull, my_d[s2], q);
      const int oi = __shfl_sync(kFull, mine[s2], q);
#pragma unroll
      for (int s = 0; s < kPer; ++s) rank[s] += before(od, oi, my_d[s], mine[s]);
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

__global__ void __launch_bounds__(256)
knn_csr_wide_rerank_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                           const float* __restrict__ vals, int64_t lo, int64_t rows,
                           const int32_t* __restrict__ cand_idx, int k, int32_t* __restrict__ out_idx,
                           float* __restrict__ out_d2) {
  csr_wide_rerank_row<kWideKK>(indptr, cols, vals, lo, rows, cand_idx, k, out_idx, out_d2);
}

// the 288 candidates of the long search, with the same merge
__global__ void __launch_bounds__(256)
knn_csr_long_rerank_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                           const float* __restrict__ vals, int64_t lo, int64_t rows,
                           const int32_t* __restrict__ cand_idx, int k, int32_t* __restrict__ out_idx,
                           float* __restrict__ out_d2) {
  csr_wide_rerank_row<kLongKK>(indptr, cols, vals, lo, rows, cand_idx, k, out_idx, out_d2);
}

}  // namespace mde

namespace {

// ---------------------------------------------------------------------------------------------------------------
// merge of a row searched in S candidate slices (mde_knn_csr_rows).  The tiles keep, per slice, the top KK of the
// slice by (approximate score, index); the full search keeps the top KK of all candidates by the same order and
// re-ranks exactly those.  Every member of the global top KK is in its own slice's top KK, so the KK smallest of the
// S KK pairs, in the order of before() (-0 == +0, ties by index, an empty slot as (+inf, INT_MAX)), are the full
// search's candidates.  Re-ranking the whole union instead could return a better list than the full search's.
// One warp per query row r stages the row's S KK pairs in shared memory, ranks each among all of them (equal pairs,
// only ever empty slots, by slot) and writes those of rank < KK to sel[r][rank], -1 for empty; the re-rank kernels
// then take sel as the full search's lists, and the certificate takes sel_val, their scores, as the full search's.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kMergeWarps = 4;

__global__ void __launch_bounds__(kMergeWarps * 32)
knn_csr_merge_kernel(int64_t rows, const int32_t* __restrict__ cand_idx, const float* __restrict__ cand_val,
                     int cands, int kk, int32_t* __restrict__ sel, float* __restrict__ sel_val) {
  extern __shared__ float s_merge[];  // per warp: scores [cands], indices [cands]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r = (int64_t)blockIdx.x * kMergeWarps + warp;
  if (r >= rows) return;
  float* sd = s_merge + (size_t)warp * 2 * cands;
  int* si = reinterpret_cast<int*>(sd + cands);
  for (int j = lane; j < cands; j += 32) {
    const int c = cand_idx[r * cands + j];
    sd[j] = c >= 0 ? cand_val[r * cands + j] : kInf;
    si[j] = c >= 0 ? c : INT_MAX;
  }
  __syncwarp();
  for (int j = lane; j < cands; j += 32) {
    const float dj = sd[j];
    const int ij = si[j];
    int rank = 0;
    for (int q = 0; q < cands; ++q) {
      const float dq = sd[q];
      const int iq = si[q];
      rank += before(dq, iq, dj, ij) || (q < j && !before(dj, ij, dq, iq));
    }
    if (rank < kk) {
      sel[r * kk + rank] = ij == INT_MAX ? -1 : ij;
      sel_val[r * kk + rank] = dj;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// certificate: is the re-ranked list of a row the k smallest (distance, index) over ALL rows?
//
// The tiles rank candidate x of query q by s(x) = fl(||x||^2~ - 2 <q, x>~): the fp32 norm (the fp64 sum rounded once)
// and the cross term of the bf16 hi / lo split accumulated in fp32.  S(x) = ||x||^2 - 2 <q, x> is its exact value, so
// ||q - x||^2 = S(x) + ||q||^2.  For every x with ||x|| <= R, |s(x) - S(x)| <= E(q), and the fp32 norm of q lies
// within E(q) of ||q||^2, with
//   E(q) = sigma (2 (a_cross |q| R + eta (|q| + R)) + a_norm R^2 + a_abs),
//   a_cross  the split (the dropped lo x lo term and the split residuals, 3.1 2^-16), the fp32 accumulation of
//            m = 3 nnz(q) products (2 u per addition, u = 2^-24, allowing truncating tensor-core adds; a product with a
//            zero element of q is an exact zero, and adding an exact zero adds no error) and the score's fma (u),
//   eta      bf16 subnormals of the split, flushed or not: 2^-126 sqrt(nnz(q)) (an absolute error per element),
//   a_norm   the fp64 sum of at most d squares and its fp32 rounding (u + (d + 6) 2^-53) and the score's fma (u),
//   a_abs    underflow: 2^-126 per product, 2^-149 per norm,
// and sigma = 2, a safety factor for second-order terms (tests/test_knn_csr_offset_cpu.py derives the bound).  None of
// these depends on d through the products, so a row of a 10^5-feature matrix certifies as one of 100 features does.
//
// R need not cover every row: a row x can enter the list only if its fp32 distance is at most d2_k, the k-th re-ranked
// one, so that ||x|| <= ||q|| + ||q - x|| <= R = sqrt((qn + 2^-149) / (1 - a_norm)) + sqrt((d2_k + 2^-149) /
// (1 - delta)) (qn: the fp32 norm of q; slack 2^-40 for the fp64 arithmetic).  A few long rows elsewhere in the matrix
// therefore cost nothing, and R^2 < 2^125 keeps every score of a row within R finite (otherwise the row fails).
//
// Every row the tiles did not keep scored at least t, the KK-th kept score (+inf when the list was never filled:
// every row was kept).  A search in S candidate slices takes t from the merged list, which is the full search's list,
// so both make the same decision.  A row not kept with ||x|| <= R lies at an exact distance D >= t - E + qn - E; when
// that exceeds (d2_k + 2^-149) (1 + delta) / (1 - delta), delta = u + (d + 2) 2^-53 bounding the re-rank's relative
// rounding, its fp32 distance exceeds d2_k and it cannot enter the list.  A row that fails (NaN and +inf included) is
// searched directly (knn_csr_direct_kernel); a false failure costs time only.  The uncertified rows are appended to
// rows[] (in no particular order: each is searched on its own) and counted in the header.
// ---------------------------------------------------------------------------------------------------------------
enum { kCertCount, kCertHdrWords };
constexpr double kCertSafety = 2.0;

__global__ void __launch_bounds__(256)
knn_csr_certify_kernel(const int64_t* __restrict__ indptr, const float* __restrict__ cand_val, int kk,
                       const float* __restrict__ norms, const float* __restrict__ d2_out, int k, int64_t lo,
                       int64_t rows, int d, unsigned* __restrict__ hdr, int32_t* __restrict__ uncert) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);  // of the query range
  if (row >= rows) return;
  float t = -kInf;
  for (int q = lane; q < kk; q += 32) t = fmaxf(t, cand_val[row * kk + q]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(kFull, t, o));
  if (lane) return;
  const double u = 0x1p-24, tiny = 0x1p-149;
  const double m = 3.0 * (double)(indptr[lo + row + 1] - indptr[lo + row]);
  const double a_cross = 3.1 * 0x1p-16 + 2.0 * u * m + u;
  const double eta = 0x1p-126 * sqrt(m / 3.0);
  const double a_norm = 2.0 * u + (d + 6.0) * 0x1p-53;
  const double a_abs = 2.0 * m * 0x1p-126 + 2.0 * tiny;
  const double delta = u + (d + 2.0) * 0x1p-53;
  const double qn = (double)norms[lo + row], d2k = (double)d2_out[row * k + k - 1];
  const double qa = sqrt((qn + tiny) / (1.0 - a_norm)) * (1.0 + 0x1p-40);
  const double R = qa + sqrt((d2k + tiny) / (1.0 - delta)) * (1.0 + 0x1p-40);
  const double E = kCertSafety * (2.0 * (a_cross * qa * R + eta * (qa + R)) + a_norm * R * R + a_abs);
  const double lhs = (d2k + tiny) * (1.0 + delta) / (1.0 - delta) - qn + E;
  if (!(lhs < (double)t - E) || !(R * R < 0x1p125))
    uncert[atomicAdd(reinterpret_cast<int*>(hdr + kCertCount), 1)] = (int32_t)row;
}

// ---------------------------------------------------------------------------------------------------------------
// direct search of the uncertified rows (row r of the query range is row lo + r): one warp per row sweeps all n rows,
// 32 at a time, one candidate per lane, with the re-rank's merge_dist2 (a function of the unordered pair: the re-rank's
// bits), and keeps the k smallest (distance, index) pairs, ascending.  Only pairs up to the re-rank's k-th pair can
// belong (the re-rank's k rows are k candidates with these very distances), which keeps insertions rare.
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
knn_csr_direct_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                      const float* __restrict__ vals, int64_t n, int k, int64_t lo,
                      const unsigned* __restrict__ hdr, const int32_t* __restrict__ uncert,
                      int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  __shared__ float s_d[8][kLongMaxK];
  __shared__ int s_i[8][kLongMaxK];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t slot = (int64_t)blockIdx.x * 8 + warp;
  if (slot >= (int64_t)hdr[kCertCount]) return;
  const int64_t row = uncert[slot], q = lo + row;
  float* ld = s_d[warp];
  int* li = s_i[warp];
  for (int j = lane; j < k; j += 32) { ld[j] = kInf; li[j] = INT_MAX; }
  __syncwarp();
  const float bd = out_d2[row * k + k - 1];
  const int bi = out_idx[row * k + k - 1];
  float thr = kInf;
  int thi = INT_MAX, worst = 0;
  for (int64_t c0 = 0; c0 < n; c0 += 32) {
    const int64_t c = c0 + lane;
    float dist = kInf;
    // at most the re-rank's k-th pair
    bool offer = c < n && c != q;
    if (offer) {
      dist = (float)merge_dist2(indptr, cols, vals, q, c);
      offer = !before(bd, bi, dist, (int)c);
    }
    // the offers of this chunk in index order, each against the worst kept pair (warp-uniform)
    for (unsigned b = __ballot_sync(kFull, offer); b; b &= b - 1) {
      const int src = __ffs(b) - 1;
      const float od = __shfl_sync(kFull, dist, src);
      const int oi = (int)(c0 + src);
      if (!before(od, oi, thr, thi)) continue;
      if (lane == 0) { ld[worst] = od; li[worst] = oi; }
      __syncwarp();
      // the new worst: the largest (distance, index, slot) of the list
      float mx = -kInf; int mi = INT_MIN, w = -1;
      for (int j = lane; j < k; j += 32) {
        if (before(mx, mi, ld[j], li[j]) || (mx == ld[j] && mi == li[j])) { mx = ld[j]; mi = li[j]; w = j; }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float om = __shfl_xor_sync(kFull, mx, o);
        const int omi = __shfl_xor_sync(kFull, mi, o), ow = __shfl_xor_sync(kFull, w, o);
        if (before(mx, mi, om, omi) || (mx == om && mi == omi && ow > w)) { mx = om; mi = omi; w = ow; }
      }
      thr = mx; thi = mi; worst = w;
      __syncwarp();
    }
  }
  // ascending by (distance, index): the rank of every slot among the k
  int rank[kLongMaxK / 32];
#pragma unroll
  for (int s = 0; s < kLongMaxK / 32; ++s) {
    const int j = lane + 32 * s;
    rank[s] = 0;
    if (j < k) for (int p = 0; p < k; ++p) rank[s] += before(ld[p], li[p], ld[j], li[j]);
  }
  __syncwarp();
#pragma unroll
  for (int s = 0; s < kLongMaxK / 32; ++s) {
    const int j = lane + 32 * s;
    if (j < k) {
      out_idx[row * k + rank[s]] = li[j];
      out_d2[row * k + rank[s]] = ld[j];
    }
  }
}

}  // namespace

namespace {

// One thread per pair (the rows of a pair are walked in column order: the same fp64 sum every run).
__global__ void __launch_bounds__(256)
pair_dist_csr_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                     const float* __restrict__ vals, int64_t n, const int64_t* __restrict__ pairs, int64_t p,
                     float* __restrict__ out, int* __restrict__ bad) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p) return;
  const int64_t a = pairs[2 * i], b = pairs[2 * i + 1];
  if (a < 0 || a >= n || b < 0 || b >= n) { atomicOr(bad, 1); return; }
  out[i] = (float)sqrt(merge_dist2(indptr, cols, vals, a, b));
}

int bits_for(uint64_t count) {  // bits needed to hold 0 .. count - 1
  int b = 0;
  while (b < 64 && (1ull << b) < count) ++b;
  return b;
}

}  // namespace

namespace mde {

int csr_sort_scratch(int64_t n, int d, int64_t nnz, size_t* bytes) {
  // CUB scratch of the two sorts (a query: no device work)
  size_t t1 = 0, t2 = 0;
  MDE_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(nullptr, t1, (const int32_t*)nullptr, (int32_t*)nullptr,
                                                         (const int32_t*)nullptr, (int32_t*)nullptr, d));
  MDE_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t2, (const uint64_t*)nullptr, (uint64_t*)nullptr,
                                               (const float*)nullptr, (float*)nullptr, (int64_t)nnz, 0,
                                               bits_for((uint64_t)n) + bits_for((uint64_t)d)));
  *bytes = t1 > t2 ? t1 : t2;
  return 0;
}

size_t csr_sort_scratch_bound(int d, int64_t nnz) {
  const size_t items = (size_t)(nnz > (int64_t)d ? nnz : (int64_t)d);
  return 16 * items + (8u << 20);
}

int csr_knn_layout(int64_t n, int d, int64_t nnz, CsrKnnLayout* L, int kk) {
  size_t tmp = 0;
  const int rc = csr_sort_scratch(n, d, nnz, &tmp);
  if (rc) return rc;
  csr_knn_carve(n, d, nnz, kk, tmp, L);
  return 0;
}

void csr_knn_carve(int64_t n, int d, int64_t nnz, int kk, size_t tmp_bytes, CsrKnnLayout* L) {
  L->n_pad = (n + kTileN - 1) / kTileN * kTileN;
  L->num_tiles = (int)(L->n_pad / kTileN);
  const int64_t nkb = ((int64_t)d + kBlockK - 1) / kBlockK;
  L->nwords = (int)((nkb + 31) / 32);
  L->row_bits = bits_for((uint64_t)n);
  L->col_bits = bits_for((uint64_t)d);
  L->tmp_bytes = tmp_bytes;
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  size_t o = 0;
  L->off_flag = o; o = up(o + 4);
  L->off_norm = o; o = up(o + (size_t)L->n_pad * 4);
  L->off_ci = o; o = up(o + (size_t)n * kk * 4);
  L->off_cv = o; o = up(o + (size_t)n * kk * 4);
  L->off_cnt = o; o = up(o + (size_t)d * 4);
  L->off_cnt_s = o; o = up(o + (size_t)d * 4);
  L->off_iota = o; o = up(o + (size_t)d * 4);
  L->off_col_s = o; o = up(o + (size_t)d * 4);
  L->off_perm = o; o = up(o + (size_t)d * 4);
  L->off_bm = o; o = up(o + (size_t)L->num_tiles * L->nwords * 4);
  L->off_kin = o; o = up(o + (size_t)nnz * 8);  // after the sort: the re-sorted column indices (int32)
  L->off_kout = o; o = up(o + (size_t)nnz * 8);
  L->off_val = o; o = up(o + (size_t)nnz * 4);
  L->off_tmp = o; o = up(o + L->tmp_bytes);
  L->off_hdr = L->off_rows = 0;
  if (kk > 0) {
    L->off_hdr = o; o = up(o + 4 * kCertHdrWords);  // the certificate's header
    L->off_rows = o; o = up(o + (size_t)n * 4);     // the uncertified rows
  }
  L->total = o;
}

}  // namespace mde

namespace {

// Runs csr_check_kernel and reads the verdict back (blocking).
int check_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
              int64_t n_pad, int* flag_dev, int32_t* col_count, float* norms, cudaStream_t st) {
  MDE_CUDA_TRY(cudaMemsetAsync(flag_dev, 0, sizeof(int), st));
  csr_check_kernel<<<(unsigned)((n_pad + 7) / 8), 256, 0, st>>>(indptr, indices, values, n, d, nnz, n_pad, flag_dev,
                                                              col_count, norms);
  MDE_LAUNCH_CHECK();
  int flag = 0;
  MDE_CUDA_TRY(cudaMemcpyAsync(&flag, flag_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  return flag ? MDE_E_INVALID : 0;
}

}  // namespace

namespace mde {

int prepare_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                const CsrKnnLayout& L, uint8_t* w, cudaStream_t st) {
  int* flag = reinterpret_cast<int*>(w + L.off_flag);
  float* norms = reinterpret_cast<float*>(w + L.off_norm);
  int32_t* cnt = reinterpret_cast<int32_t*>(w + L.off_cnt);
  int32_t* cnt_s = reinterpret_cast<int32_t*>(w + L.off_cnt_s);
  int32_t* iota = reinterpret_cast<int32_t*>(w + L.off_iota);
  int32_t* col_s = reinterpret_cast<int32_t*>(w + L.off_col_s);
  int32_t* perm = reinterpret_cast<int32_t*>(w + L.off_perm);
  uint32_t* bm = reinterpret_cast<uint32_t*>(w + L.off_bm);
  uint64_t* kin = reinterpret_cast<uint64_t*>(w + L.off_kin);
  uint64_t* kout = reinterpret_cast<uint64_t*>(w + L.off_kout);
  int32_t* cols = reinterpret_cast<int32_t*>(w + L.off_kin);
  float* vals = reinterpret_cast<float*>(w + L.off_val);
  void* tmp = w + L.off_tmp;
  size_t tmp_bytes = L.tmp_bytes;

  MDE_CUDA_TRY(cudaMemsetAsync(cnt, 0, (size_t)d * 4, st));
  int rc;
  if ((rc = check_csr(indptr, indices, values, n, d, nnz, L.n_pad, flag, cnt, norms, st))) return rc;
  // features by descending document frequency (stable: equal counts keep column order)
  iota_kernel<<<(d + 255) / 256, 256, 0, st>>>(iota, d);
  MDE_LAUNCH_CHECK();
  MDE_CUDA_TRY(cub::DeviceRadixSort::SortPairsDescending(tmp, tmp_bytes, cnt, cnt_s, iota, col_s, d, 0, 32, st));
  invert_perm_kernel<<<(d + 255) / 256, 256, 0, st>>>(col_s, d, perm);
  MDE_LAUNCH_CHECK();
  MDE_CUDA_TRY(cudaMemsetAsync(bm, 0, (size_t)L.num_tiles * L.nwords * 4, st));
  if (nnz > 0) {
    csr_keys_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(indptr, indices, perm, n, L.col_bits, L.nwords, kin, bm);
    MDE_LAUNCH_CHECK();
    tmp_bytes = L.tmp_bytes;
    MDE_CUDA_TRY(cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, kin, kout, values, vals, (int64_t)nnz, 0,
                                                 L.row_bits + L.col_bits, st));
    key_to_col_kernel<<<(unsigned)((nnz + 255) / 256), 256, 0, st>>>(kout, nnz, (1ull << L.col_bits) - 1, cols);
    MDE_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace mde

namespace {

// The tile shape of a search: tm query rows per CTA, tn candidates per tile, kk candidates kept per row.
struct CsrShape { int tm, tn, kk; };
constexpr CsrShape kCsrNarrow{kTileM, kTileN, kKK}, kCsrWide{kWideTileM, kTileN, kWideKK},
    kCsrLong{kWideTileM, kLongTileN, kLongKK};

CsrShape csr_shape(int k) { return k > kWideMaxK ? kCsrLong : k > kMaxK ? kCsrWide : kCsrNarrow; }

// Candidate slices of a search of `rows` query rows against the n rows (mde_logic.h: knn_slices).  The long search
// keeps one: the merge of its 288-candidate lists would not fit in shared memory.
int csr_search_slices(int64_t n, int64_t rows, CsrShape sh) {
  if (sh.kk == kLongKK) return 1;
  const int64_t n_pad = (n + kTileN - 1) / kTileN * kTileN;
  return knn_slices((rows + sh.tm - 1) / sh.tm, n_pad / sh.tn, kNumSMs, kMaxSlices);
}

// mde_knn_csr_rows: prepare_csr's workspace (without candidate lists, its sort scratch reserved as
// csr_sort_scratch_bound, so that the size is host arithmetic alone), then the lists of the query rows, S per row,
// the KK candidates per row the merge selects with their scores, and the certificate's header and row ids.  The lists take room for rows, or, when the rule may split, the
// most a split can hold (q_tiles S <= kNumSMs, S <= kMaxSlices): a workspace sized for a search fits every search of
// fewer rows, and grows with n.
struct CsrRowsLayout {
  CsrKnnLayout prep;
  int slices;
  size_t off_ci, off_cv, off_sel, off_selv, off_hdr, off_rows, total;
};

CsrRowsLayout csr_rows_layout(int64_t n, int d, int64_t nnz, int64_t rows, CsrShape sh) {
  CsrRowsLayout R;
  csr_knn_carve(n, d, nnz, 0, csr_sort_scratch_bound(d, nnz), &R.prep);
  R.slices = csr_search_slices(n, rows, sh);
  int64_t cap = rows;
  if (sh.kk != kLongKK) {
    const int64_t split = rows * kMaxSlices < (int64_t)kNumSMs * sh.tm ? rows * kMaxSlices : (int64_t)kNumSMs * sh.tm;
    if (split > cap) cap = split;
  }
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  size_t o = R.prep.total;
  R.off_ci = o; o = up(o + (size_t)cap * sh.kk * 4);
  R.off_cv = o; o = up(o + (size_t)cap * sh.kk * 4);
  R.off_sel = o; o = up(o + (size_t)rows * sh.kk * 4);
  R.off_selv = o; o = up(o + (size_t)rows * sh.kk * 4);     // their scores, for the certificate
  R.off_hdr = o; o = up(o + 4 * kCertHdrWords);             // the certificate's header
  R.off_rows = o; o = up(o + (size_t)rows * 4);             // the uncertified rows
  R.total = o;
  return R;
}

// The prepared rows and the bitmaps of a workspace laid out by L.
struct CsrPrepared {
  const float* norms;
  const uint32_t* bm;
  const int32_t* cols;
  const float* vals;
};

CsrPrepared prepared(const CsrKnnLayout& L, const uint8_t* w) {
  return {reinterpret_cast<const float*>(w + L.off_norm), reinterpret_cast<const uint32_t*>(w + L.off_bm),
          reinterpret_cast<const int32_t*>(w + L.off_kin), reinterpret_cast<const float*>(w + L.off_val)};
}

// The tiles of the query range qr (one CTA per query tile and candidate slice) into lists of sh.kk per row and slice.
int launch_tiles(CsrShape sh, const int64_t* indptr, const CsrPrepared& P, const CsrKnnLayout& L, int64_t n,
                 const QueryRange& qr, int32_t* ci, float* cv, cudaStream_t st) {
  const dim3 grid((unsigned)((qr.hi - qr.base + sh.tm - 1) / sh.tm), (unsigned)qr.slices);
  const int num_tiles = (int)(L.n_pad / sh.tn);
  if (sh.kk == kKK) {
    static bool attr_set = false;
    if (!attr_set) {
      MDE_CUDA_TRY(cudaFuncSetAttribute(knn_csr_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
      attr_set = true;
    }
    knn_csr_tile_kernel<<<grid, kThreads, kSmemBytes, st>>>(indptr, P.cols, P.vals, P.norms, P.bm, L.nwords, n,
                                                            num_tiles, qr, ci, cv);
  } else if (sh.kk == kWideKK) {
    constexpr int kSmem = kWideSmemBytes<kWideKK, kTileN>;
    static bool attr_set = false;
    if (!attr_set) {
      MDE_CUDA_TRY(cudaFuncSetAttribute(knn_csr_wide_tile_kernel<kWideKK, kTileN>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
      attr_set = true;
    }
    knn_csr_wide_tile_kernel<kWideKK, kTileN><<<grid, 2 * kTileN, kSmem, st>>>(indptr, P.cols, P.vals, P.norms, P.bm,
                                                                              L.nwords, n, num_tiles, qr, ci, cv);
  } else {
    constexpr int kSmem = kWideSmemBytes<kLongKK, kLongTileN>;
    static bool attr_set = false;
    if (!attr_set) {
      MDE_CUDA_TRY(cudaFuncSetAttribute(knn_csr_wide_tile_kernel<kLongKK, kLongTileN>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
      attr_set = true;
    }
    knn_csr_wide_tile_kernel<kLongKK, kLongTileN><<<grid, 2 * kLongTileN, kSmem, st>>>(
        indptr, P.cols, P.vals, P.norms, P.bm, L.nwords, n, num_tiles, qr, ci, cv);
  }
  MDE_LAUNCH_CHECK();
  return 0;
}

// The exact re-rank of kk candidates per query row lo + r, 0 <= r < rows, into the compact outputs [rows][k].
int launch_rerank(int kk, const int64_t* indptr, const CsrPrepared& P, int64_t lo, int64_t rows, const int32_t* ci,
                  int k, int32_t* idx_out, float* d2_out, cudaStream_t st) {
  const unsigned grid = (unsigned)((rows + 7) / 8);
  if (kk == kKK)
    knn_csr_rerank_kernel<<<grid, 256, 0, st>>>(indptr, P.cols, P.vals, lo, rows, ci, k, idx_out, d2_out);
  else if (kk == kWideKK)
    knn_csr_wide_rerank_kernel<<<grid, 256, 0, st>>>(indptr, P.cols, P.vals, lo, rows, ci, k, idx_out, d2_out);
  else
    knn_csr_long_rerank_kernel<<<grid, 256, 0, st>>>(indptr, P.cols, P.vals, lo, rows, ci, k, idx_out, d2_out);
  MDE_LAUNCH_CHECK();
  return 0;
}

// After the re-rank of the query rows lo + r, 0 <= r < rows: certify every row against its kk kept scores cv[r][.],
// search the uncertified rows directly; with `fallback_rows`, wait for the stream and report how many rows that was.
int certify_direct(const int64_t* indptr, const CsrPrepared& P, int64_t n, int d, int64_t lo, int64_t rows, int kk,
                   const float* cv, int k, int32_t* idx_out, float* d2_out, unsigned* hdr, int32_t* uncert,
                   cudaStream_t st, int* fallback_rows) {
  MDE_CUDA_TRY(cudaMemsetAsync(hdr, 0, 4 * kCertHdrWords, st));
  const unsigned grid = (unsigned)((rows + 7) / 8);
  knn_csr_certify_kernel<<<grid, 256, 0, st>>>(indptr, cv, kk, P.norms, d2_out, k, lo, rows, d, hdr, uncert);
  MDE_LAUNCH_CHECK();
  knn_csr_direct_kernel<<<grid, 256, 0, st>>>(indptr, P.cols, P.vals, n, k, lo, hdr, uncert, idx_out, d2_out);
  MDE_LAUNCH_CHECK();
  if (fallback_rows) {
    MDE_CUDA_TRY(cudaMemcpyAsync(fallback_rows, hdr + kCertCount, sizeof(int), cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaStreamSynchronize(st));
  }
  return 0;
}

bool bad_csr_args(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                  int k, int max_k, const void* idx_out, const void* d2_out, const void* ws) {
  return !indptr || !idx_out || !d2_out || !ws || n < 2 || d < 1 || nnz < 0 || k < 1 || k > max_k || k > n - 1 ||
         (nnz > 0 && (!indices || !values));
}

int csr_full_ws_bytes(int64_t n, int d, int64_t nnz, int kk, size_t* bytes) {
  if (!bytes || n < 2 || d < 1 || nnz < 0) return MDE_E_INVALID;
  CsrKnnLayout L;
  int rc = csr_knn_layout(n, d, nnz, &L, kk);
  if (rc) return rc;
  *bytes = L.total;
  return 0;
}

// mde_knn_csr (k <= 24), mde_knn_csr_wide (k <= 64), mde_knn_csr_long (k <= 256): prep, the tiles of [0, n) in one
// slice, re-rank of all KK candidates of every row.
int run_csr_full(CsrShape sh, const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                 int64_t nnz, int k, int max_k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
                 void* stream, int* fallback_rows) {
  if (bad_csr_args(indptr, indices, values, n, d, nnz, k, max_k, idx_out, d2_out, ws)) return MDE_E_INVALID;
  if (n > (1ll << 31) - kTileN) return MDE_E_UNSUPPORTED;
  CsrKnnLayout L;
  int rc = csr_knn_layout(n, d, nnz, &L, sh.kk);
  if (rc) return rc;
  if (ws_bytes < L.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = static_cast<uint8_t*>(ws);
  if ((rc = prepare_csr(indptr, indices, values, n, d, nnz, L, w, st))) return rc;
  const CsrPrepared P = prepared(L, w);
  int32_t* ci = reinterpret_cast<int32_t*>(w + L.off_ci);
  float* cv = reinterpret_cast<float*>(w + L.off_cv);
  if ((rc = launch_tiles(sh, indptr, P, L, n, QueryRange{0, 0, n, 1}, ci, cv, st))) return rc;
  if ((rc = launch_rerank(sh.kk, indptr, P, 0, n, ci, k, idx_out, d2_out, st))) return rc;
  return certify_direct(indptr, P, n, d, 0, n, sh.kk, cv, k, idx_out, d2_out,
                        reinterpret_cast<unsigned*>(w + L.off_hdr), reinterpret_cast<int32_t*>(w + L.off_rows), st,
                        fallback_rows);
}

// mde_knn_csr_rows: prep of the whole matrix, the tiles of the query tiles only (in S candidate slices), the merge
// of the S lists of a row when S > 1, re-rank.  Query tiles keep the full search's alignment (base: lo rounded down
// to sh.tm), so that every (query tile, candidate tile) pair, and with it every score, is the full search's.
int run_csr_rows(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                 int64_t lo, int64_t hi, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
                 void* stream, int* fallback_rows) {
  if (bad_csr_args(indptr, indices, values, n, d, nnz, k, kLongMaxK, idx_out, d2_out, ws) || lo < 0 || hi > n ||
      lo >= hi)
    return MDE_E_INVALID;
  if (n > (1ll << 31) - kTileN) return MDE_E_UNSUPPORTED;
  const CsrShape sh = csr_shape(k);
  const int64_t rows = hi - lo;
  const CsrRowsLayout R = csr_rows_layout(n, d, nnz, rows, sh);
  if (ws_bytes < R.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  size_t sort_bytes = 0;
  int rc = csr_sort_scratch(n, d, nnz, &sort_bytes);
  if (rc) return rc;
  if (sort_bytes > R.prep.tmp_bytes) return MDE_E_ALLOC;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = static_cast<uint8_t*>(ws);
  if ((rc = prepare_csr(indptr, indices, values, n, d, nnz, R.prep, w, st))) return rc;
  const CsrPrepared P = prepared(R.prep, w);
  int32_t* ci = reinterpret_cast<int32_t*>(w + R.off_ci);
  float* cv = reinterpret_cast<float*>(w + R.off_cv);
  const QueryRange qr{lo / sh.tm * sh.tm, lo, hi, R.slices};
  if ((rc = launch_tiles(sh, indptr, P, R.prep, n, qr, ci, cv, st))) return rc;
  const int32_t* lists = ci;
  const float* scores = cv;
  if (R.slices > 1) {
    int32_t* sel = reinterpret_cast<int32_t*>(w + R.off_sel);
    float* sel_val = reinterpret_cast<float*>(w + R.off_selv);
    const int cands = R.slices * sh.kk;
    knn_csr_merge_kernel<<<(unsigned)((rows + kMergeWarps - 1) / kMergeWarps), kMergeWarps * 32,
                           (size_t)kMergeWarps * cands * 8, st>>>(rows, ci, cv, cands, sh.kk, sel, sel_val);
    MDE_LAUNCH_CHECK();
    lists = sel;
    scores = sel_val;
  }
  if ((rc = launch_rerank(sh.kk, indptr, P, lo, rows, lists, k, idx_out, d2_out, st))) return rc;
  return certify_direct(indptr, P, n, d, lo, rows, sh.kk, scores, k, idx_out, d2_out,
                        reinterpret_cast<unsigned*>(w + R.off_hdr), reinterpret_cast<int32_t*>(w + R.off_rows), st,
                        fallback_rows);
}

}  // namespace

extern "C" {

int mde_knn_csr_ws_bytes(int64_t n, int d, int64_t nnz, size_t* bytes) {
  return csr_full_ws_bytes(n, d, nnz, kKK, bytes);
}

int mde_knn_csr_ex(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                   int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream,
                   int* fallback_rows) {
  return run_csr_full(kCsrNarrow, indptr, indices, values, n, d, nnz, k, kMaxK, idx_out, d2_out, ws, ws_bytes,
                      stream, fallback_rows);
}

int mde_knn_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream) {
  return mde_knn_csr_ex(indptr, indices, values, n, d, nnz, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_csr_wide_ws_bytes(int64_t n, int d, int64_t nnz, size_t* bytes) {
  return csr_full_ws_bytes(n, d, nnz, kWideKK, bytes);
}

int mde_knn_csr_wide_ex(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                        int64_t nnz, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream,
                        int* fallback_rows) {
  return run_csr_full(kCsrWide, indptr, indices, values, n, d, nnz, k, kWideMaxK, idx_out, d2_out, ws, ws_bytes,
                      stream, fallback_rows);
}

int mde_knn_csr_wide(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                     int64_t nnz, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream) {
  return mde_knn_csr_wide_ex(indptr, indices, values, n, d, nnz, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_csr_long_ws_bytes(int64_t n, int d, int64_t nnz, size_t* bytes) {
  return csr_full_ws_bytes(n, d, nnz, kLongKK, bytes);
}

int mde_knn_csr_long_ex(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                        int64_t nnz, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream,
                        int* fallback_rows) {
  return run_csr_full(kCsrLong, indptr, indices, values, n, d, nnz, k, kLongMaxK, idx_out, d2_out, ws, ws_bytes,
                      stream, fallback_rows);
}

int mde_knn_csr_long(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                     int64_t nnz, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream) {
  return mde_knn_csr_long_ex(indptr, indices, values, n, d, nnz, k, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_csr_rows_ws_bytes(int64_t n, int d, int64_t nnz, int64_t rows, int k, size_t* bytes) {
  if (!bytes || n < 2 || d < 1 || nnz < 0 || rows < 1 || rows > n || k < 1 || k > kLongMaxK || k > n - 1)
    return MDE_E_INVALID;
  *bytes = csr_rows_layout(n, d, nnz, rows, csr_shape(k)).total;
  return 0;
}

int mde_knn_csr_rows_ex(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                        int64_t nnz, int64_t row_begin, int64_t row_end, int k, int32_t* idx_out, float* d2_out,
                        void* ws, size_t ws_bytes, void* stream, int* fallback_rows) {
  return run_csr_rows(indptr, indices, values, n, d, nnz, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes,
                      stream, fallback_rows);
}

int mde_knn_csr_rows(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                     int64_t nnz, int64_t row_begin, int64_t row_end, int k, int32_t* idx_out, float* d2_out, void* ws,
                     size_t ws_bytes, void* stream) {
  return mde_knn_csr_rows_ex(indptr, indices, values, n, d, nnz, row_begin, row_end, k, idx_out, d2_out, ws, ws_bytes,
                             stream, nullptr);
}

// host-side debug entry point: the candidate slices (mde_logic.h: knn_slices) of mde_knn_csr_rows for `rows` query
// rows against n rows with k neighbours (narrow tiles up to k = 24, wide up to 64, long, in one slice, up to 256);
// -1 for bad arguments
int mde_dbg_knn_csr_slices(int64_t n, int64_t rows, int k) {
  if (n < 2 || rows < 1 || rows > n || k < 1 || k > kLongMaxK) return -1;
  return csr_search_slices(n, rows, csr_shape(k));
}

int mde_pair_dist_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                      const int64_t* pairs, int64_t p, float* out, void* stream) {
  if (!indptr || n < 1 || d < 1 || p < 0 || (p > 0 && (!pairs || !out))) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  int64_t nnz = 0;
  MDE_CUDA_TRY(cudaMemcpyAsync(&nnz, indptr + n, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  if (nnz < 0 || (nnz > 0 && (!indices || !values))) return MDE_E_INVALID;
  int* flag = nullptr;
  MDE_CUDA_TRY(cudaMallocAsync(reinterpret_cast<void**>(&flag), sizeof(int), st));
  int rc = check_csr(indptr, indices, values, n, d, nnz, n, flag, nullptr, nullptr, st);
  if (!rc && p > 0) {
    pair_dist_csr_kernel<<<(unsigned)((p + 255) / 256), 256, 0, st>>>(indptr, indices, values, n, pairs, p, out, flag);
    MDE_LAUNCH_CHECK();
    int bad = 0;
    MDE_CUDA_TRY(cudaMemcpyAsync(&bad, flag, sizeof(int), cudaMemcpyDeviceToHost, st));
    MDE_CUDA_TRY(cudaStreamSynchronize(st));
    if (bad) rc = MDE_E_INVALID;
  }
  MDE_CUDA_TRY(cudaFreeAsync(flag, st));
  return rc;
}

}  // extern "C"
