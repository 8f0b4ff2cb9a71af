// mde_knn_csr.cuh -- what the exact (mde_knn_sparse.cu) and the approximate (mde_knn_approx.cu) k-nearest-neighbour
// searches of a CSR data matrix share: the preparation of the rows, the exact pair distance and the re-rank kernels.
// Both searches measure every pair with merge_dist2 over the rows as prepare_csr re-sorts them, so a pair found by
// both carries the same fp32 bits.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "mde_knn_select.cuh"

namespace mde {

// Workspace of the preparation (and of the exact searches' candidate lists, kk per row, and their certificate: a
// header and n row ids, at the end), 1024-byte aligned offsets.
struct CsrKnnLayout {
  int64_t n_pad; int num_tiles, nwords, row_bits, col_bits;
  size_t off_flag, off_norm, off_ci, off_cv, off_cnt, off_cnt_s, off_iota, off_col_s, off_perm, off_bm, off_kin,
      off_kout, off_val, off_tmp, tmp_bytes, off_hdr, off_rows, total;
};

// Scratch bytes of the two CUB radix sorts of prepare_csr: a query that needs a device but does no device work.
int csr_sort_scratch(int64_t n, int d, int64_t nnz, size_t* bytes);
// A bound on that scratch in host arithmetic alone, for workspace queries that must not need a device: 16 bytes per
// item of the larger sort (the alternate key and value buffers take 12, CUB's look-back at most 4) plus 8 MB of
// histograms.  A search sized by it checks csr_sort_scratch against it before it starts.
size_t csr_sort_scratch_bound(int d, int64_t nnz);
// The layout for a given sort scratch (host arithmetic only).  kk: candidates kept per row (kNarrowKK, or kWideKK for
// the wide search; 0 when the caller keeps its own lists, and its own certificate state, elsewhere).
void csr_knn_carve(int64_t n, int d, int64_t nnz, int kk, size_t tmp_bytes, CsrKnnLayout* L);
// csr_knn_carve with the scratch csr_sort_scratch reports.
int csr_knn_layout(int64_t n, int d, int64_t nnz, CsrKnnLayout* L, int kk = kNarrowKK);

// Validates the CSR (blocking status read: MDE_E_INVALID when malformed), writes the norms, the feature permutation
// by descending document frequency, the rows re-sorted under it (column indices at off_kin, values at off_val; the
// caller's indptr still delimits them) and the per-tile occupancy bitmaps.  Uses the whole of L's workspace at w
// except off_ci / off_cv.
int prepare_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                const CsrKnnLayout& L, uint8_t* w, cudaStream_t st);

// sum (a_f - b_f)^2 over two rows given as (sorted columns, values, length), merged in column order, in fp64.  Each
// term depends on one column alone and the columns are visited in the same order whichever row comes first, so the
// sum is a function of the unordered pair.  The pointers may address global or shared memory.
__device__ __forceinline__ double merge_dist2_rows(const int32_t* __restrict__ ca, const float* __restrict__ va,
                                                   int na, const int32_t* __restrict__ cb,
                                                   const float* __restrict__ vb, int nb) {
  int p = 0, q = 0;
  double acc = 0.0;
  while (p < na && q < nb) {
    const int cp = ca[p], cq = cb[q];
    double t;
    if (cp == cq) { t = (double)va[p] - (double)vb[q]; ++p; ++q; }
    else if (cp < cq) { t = va[p]; ++p; }
    else { t = vb[q]; ++q; }
    acc = fma(t, t, acc);
  }
  for (; p < na; ++p) { const double t = va[p]; acc = fma(t, t, acc); }
  for (; q < nb; ++q) { const double t = vb[q]; acc = fma(t, t, acc); }
  return acc;
}

// The same sum for rows a and b of a validated CSR (row lengths are below d < 2^31).
__device__ __forceinline__ double merge_dist2(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                                              const float* __restrict__ vals, int64_t a, int64_t b) {
  const int64_t pa = indptr[a], pb = indptr[b];
  return merge_dist2_rows(cols + pa, vals + pa, (int)(indptr[a + 1] - pa), cols + pb, vals + pb,
                          (int)(indptr[b + 1] - pb));
}

// (float)merge_dist2 of a row's kNarrowKK (knn_csr_rerank_kernel) or kWideKK (knn_csr_wide_rerank_kernel) candidates
// cand_idx[r][.], -1 for none, for the query rows lo + r, 0 <= r < rows; the k smallest by (distance, index) go to
// out_idx / out_d2 [rows][k] in ascending order.  One warp per row, 256 threads per block.
__global__ void __launch_bounds__(256)
knn_csr_rerank_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                      const float* __restrict__ vals, int64_t lo, int64_t rows, const int32_t* __restrict__ cand_idx,
                      int k, int32_t* __restrict__ out_idx, float* __restrict__ out_d2);
__global__ void __launch_bounds__(256)
knn_csr_wide_rerank_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                           const float* __restrict__ vals, int64_t lo, int64_t rows,
                           const int32_t* __restrict__ cand_idx, int k, int32_t* __restrict__ out_idx,
                           float* __restrict__ out_d2);

}  // namespace mde
