// mde_project.cuh -- constraint projections shared by the C ABI (mde_project.cu) and the
// solver (mde_solver.cu).  Reference: pymde/constraints.py:94-200, pymde/util.py:129-171.
#pragma once
#include "mde_common.cuh"

namespace mde {

constexpr int kProjMaxM = 32;    // Standardized, narrow rows: m <= 32 (Gram + warp Jacobi in one block)
constexpr int kWideMaxM = 1024;  // Standardized, wide rows: 32 < m <= 1024 (tiled Gram, Newton-Schulz inverse square root)
constexpr int kWideTileM = 256;  // m <= 256: 64 x 64 Gram tiles and FFMA Newton-Schulz products; above, 128 x 128 and DMMA
constexpr int kWideRowBlocks = 2 * kNumSMs;  // row blocks of the tiled Gram kernel (target: tiles^2 x row blocks)
// Fewest row blocks of the tiled Gram: each block sums at most ceil(n / 16) rows in one fp32 run, the length m = 256
// reaches with kWideRowBlocks / 4^2 = 16 blocks, whatever the width.
constexpr int kWideMinRowBlocks = 16;
constexpr int kWideNsIters = 24; // gated Newton-Schulz iterations enqueued per retraction
constexpr int kProjBlocks = kNumSMs * 2;
constexpr int kProjThreads = 256;
// The narrow retraction reports a Gram whose smallest eigenvalue is <= kProjRankTol * the largest as singular.
constexpr double kProjRankTol = 1e-12;

// The Standardized retraction takes its Gram of X - s.  s[c] = X[0][c] + the fp32 mean of X[r][c] - X[0][c] over the
// first min(n, kShiftRows) rows: close to the column mean whether or not X is centred (X[0] alone would add n s s^T
// of the order of the spread to an already centred Gram), and exactly X[0][c] for a constant column.  Every thread
// that needs s[c] computes it with the same operations, so all of a launch agree.
constexpr int kShiftRows = 32;
__device__ __forceinline__ float proj_shift(const float* X, int64_t n, int m, int c) {
  const int k = n < kShiftRows ? (int)n : kShiftRows;
  const float x0 = X[c];
  float a = 0.0f;
  for (int r = 1; r < k; ++r) a += X[(int64_t)r * m + c] - x0;
  return x0 + a / (float)k;
}

// workspace (doubles): [0, kProjBlocks * K) block partials, then finals
struct ProjWs {
  double* partials;  // kProjBlocks * kmax
  double* mean;      // m            (column means)
  double* shift;     // m            (proj_shift of the retracted X: its Gram is taken of X - shift)
  double* mat;       // m*m          (W for the retraction, or Z^T X / n for the tangent)
  int* status;       // 1 int, written by every Standardized retraction: 0 ok, 1 = the de-meaned X is (numerically)
                     // rank deficient -- n <= m, a singular Gram, or a Newton-Schulz chain that did not converge
  // ---- wide rows (32 < m <= kWideMaxM), null otherwise; in this order after status + 8 doubles ----
  float* fpart;      // row_blocks x m*m fp32 partial Gram
  double* gram;      // m*m   Z^T X (or X^T X)
  double* ns;        // 5 x m*m: Y0, Y1, Z0, Z1, T of the coupled Newton-Schulz iteration
  float* wf;         // m*m   fp32 matrix the row kernel multiplies by
  double* scal;      // [0] c (scaling), [1..3] residual slots of the Newton-Schulz iterations (it % 3)
  int* nsflag;       // [0] converged (sticky), [1] buffer holding the final Z
};

inline int64_t proj_mm(int m) { return m <= kProjMaxM ? (int64_t)m * m : 0; }

inline bool proj_wide(int m) { return m > kProjMaxM && m <= kWideMaxM; }
// output tile of the tiled Gram kernel: 64 x 64 up to m = 256, 128 x 128 above
inline int wide_gram_tile(int m) { return m <= kWideTileM ? 64 : 128; }
// row blocks of the tiled Gram kernel for width m (the grid is tiles^2 x row blocks): 264 / tiles^2, at least 16
// (which leaves every m <= 256 as it was: 264 / 4^2 = 16).
inline int wide_row_blocks(int m) {
  const int t = wide_gram_tile(m);
  const int tiles = (m + t - 1) / t;
  const int rb = kWideRowBlocks / (tiles * tiles);
  return rb < kWideMinRowBlocks ? kWideMinRowBlocks : rb;
}
// fp32 partial Gram floats: row blocks x m^2.  Above m = 256 the region is max(16 m^2, 264 x 128^2), which holds
// every launch (264 / tiles^2 row blocks of tiles^2 128 x 128 tiles, or 16 row blocks of m^2) and grows with m:
// 16.5 MiB up to m = 519, 64 MiB at m = 1024.
inline int64_t wide_fpart_floats(int m) {
  const int64_t mm = (int64_t)m * m;
  if (m <= kWideTileM) return (int64_t)wide_row_blocks(m) * mm;
  const int64_t a = (int64_t)kWideMinRowBlocks * mm, b = (int64_t)kWideRowBlocks * 128 * 128;
  return a > b ? a : b;
}

// Workspace layout, in doubles from the start (K = m + proj_mm(m), mm = m * m):
//   partials  kProjBlocks * K
//   mean      m
//   shift     m
//   mat       proj_mm(m)
//   status    8            (one int used)
//   wide rows only:
//   fpart     wide_fpart_floats(m) / 2 + 1      (fp32)
//   gram      mm
//   ns        5 * mm
//   wf        mm / 2 + 1                        (fp32)
//   scal      8
//   nsflag    2            (two ints used)
// mde_project_ws_bytes adds 64 bytes.  At m = 1024: 64 MiB of fpart, 52 MiB of gram, ns and wf, 118.1 MiB in all.
inline int64_t proj_ws_doubles(int m) {
  int64_t k = (int64_t)m + proj_mm(m);
  int64_t base = (int64_t)kProjBlocks * k + 2 * m + proj_mm(m) + 8;
  if (proj_wide(m)) {
    const int64_t mm = (int64_t)m * m;
    base += wide_fpart_floats(m) / 2 + 1;          // fpart (floats)
    base += mm;                                    // gram
    base += 5 * mm;                                // ns
    base += mm / 2 + 1;                            // wf (floats)
    base += 8 + 2;                                 // scal, nsflag
  }
  return base;
}

inline ProjWs proj_ws_carve(void* ws, int m) {
  ProjWs w;
  int64_t k = (int64_t)m + proj_mm(m);
  w.partials = (double*)ws;
  w.mean = w.partials + (int64_t)kProjBlocks * k;
  w.shift = w.mean + m;
  w.mat = w.shift + m;
  w.status = (int*)(w.mat + proj_mm(m));
  w.fpart = nullptr; w.gram = nullptr; w.ns = nullptr; w.wf = nullptr; w.scal = nullptr; w.nsflag = nullptr;
  if (proj_wide(m)) {
    const int64_t mm = (int64_t)m * m;
    double* p = w.mat + proj_mm(m) + 8;
    w.fpart = (float*)p; p += wide_fpart_floats(m) / 2 + 1;
    w.gram = p; p += mm;
    w.ns = p; p += 5 * mm;
    w.wf = (float*)p; p += mm / 2 + 1;
    w.scal = p; p += 8;
    w.nsflag = (int*)p;
  }
  return w;
}

// Enqueue X -= colmean(X).  `active` (nullable) is a device flag; kernels exit when it is 0.
int enqueue_project_centered(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st);
// Enqueue de-mean + sqrt(n) * polar factor.  m <= kWideMaxM (1024).  Sets *w.status; nothing on the device reads it (the
// solver's in-graph retractions run on regardless), the host reads it through mde_project_status.
int enqueue_project_standardized(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st);
// Enqueue Z -= (1/n) X (Z^T X).  m <= kWideMaxM (1024).
int enqueue_tangent_standardized(const float* X, float* Z, int64_t n, int m, const ProjWs& w,
                                 const int* active, cudaStream_t st);

// wide rows (mde_project_wide.cu)
int enqueue_project_standardized_wide(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st);
int enqueue_tangent_standardized_wide(const float* X, float* Z, int64_t n, int m, const ProjWs& w,
                                      const int* active, cudaStream_t st);
// column means of a wide matrix into w.mean (mde_project.cu).  shift (nullable): summed as X - proj_shift(shift), the
// shift stored in w.shift, so that columns far from the origin keep the fp32 digits of their sums.
int enqueue_colmean_wide(const float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st,
                         const float* shift = nullptr);

}  // namespace mde
