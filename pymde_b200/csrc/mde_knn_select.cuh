// mde_knn_select.cuh -- the running top-KK lists of the wide (KK = 96, k <= 64) and long (KK = 288, k <= 256)
// k-nearest-neighbour tile kernels (mde_knn.cu, mde_knn_sparse.cu).
//
// One list of KK (distance, index) pairs per query row lives in shared memory; it is too large for registers
// next to the fp32 wgmma accumulators.  Two adjacent lanes (a "pair", half = lane & 1) own a row.  Both offer
// every candidate of the row in the same order with the same values, so both take the same branches.  The key K of a
// candidate is its fp32 score, or its exact int32 score for 8-bit input matrices (mde_knn.cu).  Lane `half`
// owns the slots of its parity: it writes the slot it replaces (when the slot is its own) and scans only its own
// slots for the new worst, and the two partial worsts meet through one shuffle.  Candidates are ordered by
// (distance, index); the worst is the largest, so the list after a sweep depends on nothing but the order of the
// offers, never on timing.
//
// It also declares the launcher of the dense re-rank kernels (defined in mde_knn.cu).  The approximate search
// (mde_knn_approx.cu) hands its final lists to them, so a pair found by the exact and the approximate search carries
// the same fp32 distance bits.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <climits>

namespace mde {

constexpr int kNarrowKK = 32;        // candidates per row read by knn_rerank_kernel
constexpr int kWideKK = 96;          // candidates kept per row before the exact re-rank
constexpr int kWideMaxK = 64;        // leaves >= 32 spare candidates for the bf16 x 3 error of the cross terms
constexpr int kLongKK = 288;         // the same margin for the long search
constexpr int kLongMaxK = 256;

template <class K>
__device__ __forceinline__ bool knn_before(K d1, int i1, K d2, int i2) {
  return d1 < d2 || (d1 == d2 && i1 < i2);
}

// The query rows of a search, [lo, hi) of the matrix, and the candidate slice of a CTA (mde_knn_rows,
// mde_knn_csr_rows).  CTA (x, y) takes the query rows base + x TM .. + TM - 1 (base: lo rounded down to a tile of the
// full search, so that every query tile is one of the full search's) against the candidate tiles
// [slice_begin(T), slice_begin(T, 1)) of the T tiles, and keeps the list of query row r at
// list(r) = (r - lo) slices + y: the S lists of a row are adjacent.  A full search is [0, n) in one slice.
struct QueryRange {
  int64_t base, lo, hi;
  int slices;
  __device__ __forceinline__ bool has(int64_t r) const { return r >= lo && r < hi; }
  __device__ __forceinline__ int64_t list(int64_t r) const { return (r - lo) * slices + blockIdx.y; }
  __device__ __forceinline__ int slice_begin(int tiles, int next = 0) const {
    return (int)((int64_t)tiles * (blockIdx.y + next) / slices);
  }
};
constexpr int kMaxSlices = 16;  // S <= 16: a merge keeps a row's S KK <= 1536 candidates in 12 KB of shared memory

// The key that orders after every candidate: +inf, or INT_MAX for integer scores (which never reach it, mde_knn.cu).
template <class K>
__device__ __forceinline__ K key_inf() { return __builtin_huge_valf(); }
template <>
__device__ __forceinline__ int key_inf<int>() { return INT_MAX; }

// Per-lane copy of its row's threshold: the worst kept pair and its slot (identical in both lanes of the pair).
template <int KK, class K = float>
struct WideList {
  // words per row list: KK + 2 = 2 (mod 32), so the 32 lanes of a warp (16 rows) hit 32 different banks
  static constexpr int kStride = KK + 2;
  static_assert(KK % 32 == 0 && kStride % 32 == 2, "lists of whole warps, conflict-free rows");

  K* d;        // this row's distances [KK] in shared memory
  int* i;      // this row's indices [KK]; INT_MAX marks an empty slot
  int half;    // 0 or 1: the parity of the slots this lane owns
  K thr;       // worst kept pair (thr, thi) in slot `worst`
  int thi, worst;

  __device__ __forceinline__ void init(K* row_d, int* row_i, int lane_half) {
    d = row_d; i = row_i; half = lane_half;
    for (int j = half; j < KK; j += 2) { d[j] = key_inf<K>(); i[j] = INT_MAX; }
    thr = key_inf<K>(); thi = INT_MAX; worst = 0;
  }

  // Keep (dist, col) if it comes before the worst kept pair.  Both lanes of the pair call this with the same
  // arguments (pair-uniform branches).
  __device__ __forceinline__ void offer(K dist, int col) {
    if (!knn_before(dist, col, thr, thi)) return;
    if ((worst & 1) == half) { d[worst] = dist; i[worst] = col; }
    K m = d[half]; int mi = i[half], w = half;
    for (int j = half + 2; j < KK; j += 2) {
      const K v = d[j]; const int vi = i[j];
      if (knn_before(m, mi, v, vi)) { m = v; mi = vi; w = j; }
    }
    const unsigned pair = 3u << ((threadIdx.x & 31) & 30);
    const K om = __shfl_xor_sync(pair, m, 1);
    const int omi = __shfl_xor_sync(pair, mi, 1), ow = __shfl_xor_sync(pair, w, 1);
    // the larger (distance, index); equal pairs (empty slots) resolve to the lower slot, so both lanes agree
    if (knn_before(m, mi, om, omi) || (!knn_before(om, omi, m, mi) && ow < w)) { m = om; mi = omi; w = ow; }
    thr = m; thi = mi; worst = w;
  }

  // This lane's slots to the row's candidate arrays (empty slots as index -1, distance key_inf).
  __device__ __forceinline__ void store(int32_t* cand_idx, K* cand_val) const {
    for (int j = half; j < KK; j += 2) {
      cand_idx[j] = i[j] == INT_MAX ? -1 : i[j];
      cand_val[j] = d[j];
    }
  }
};

// Element types of a dense data matrix: fp32, IEEE fp16, bf16, uint8 and int8.  The searches read 16-bit and 8-bit
// matrices in place and compute every distance on the fp32 value of each element, which is exact, so such a matrix X
// gives the bits of the fp32 matrix X.float().
__device__ __forceinline__ float elem_f32(float x) { return x; }
__device__ __forceinline__ float elem_f32(__half x) { return __half2float(x); }
__device__ __forceinline__ float elem_f32(__nv_bfloat16 x) { return __bfloat162float(x); }
__device__ __forceinline__ float elem_f32(uint8_t x) { return (float)x; }
__device__ __forceinline__ float elem_f32(int8_t x) { return (float)x; }
template <class T>
__device__ __forceinline__ float load_f32(const T* p) { return elem_f32(__ldg(p)); }

// Exact fp32 squared distances sum_j (q_j - x_j)^2 (lane-strided fmaf, then a butterfly) of a row's kk candidates
// cand_idx[row][.], -1 for none, kk = kNarrowKK (knn_rerank_kernel), kWideKK (knn_wide_rerank_kernel) or kLongKK
// (knn_long_rerank_kernel); the k smallest by (distance, index) go to out_idx / out_d2 [n][k] in ascending order.
// One warp per row, 256 threads per block; the elements of X are converted to fp32 as they are read.  Defined in
// mde_knn.cu for T = float, __half, __nv_bfloat16, uint8_t and int8_t.
template <class T>
int knn_dense_rerank(int kk, const T* X, int64_t n, int d, const int32_t* cand_idx, int k, int32_t* out_idx,
                     float* out_d2, cudaStream_t st);

}  // namespace mde
