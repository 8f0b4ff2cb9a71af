// mde_project.cuh -- constraint projections shared by the C ABI (mde_project.cu) and the
// solver (mde_solver.cu).  Reference: pymde/constraints.py:94-200, pymde/util.py:129-171.
#pragma once
#include "mde_common.cuh"

namespace mde {

constexpr int kProjMaxM = 32;    // Standardized, narrow rows: m <= 32 (Gram + warp Jacobi in one block)
constexpr int kWideMaxM = 256;   // Standardized, wide rows: 32 < m <= 256 (tiled Gram, Newton-Schulz inverse square root)
constexpr int kWideRowBlocks = 2 * kNumSMs;  // row blocks of the tiled Gram kernel (upper bound)
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
  // ---- wide rows (32 < m <= kWideMaxM), null otherwise ----
  float* fpart;      // row_blocks x m*m fp32 partial Gram
  double* gram;      // m*m   Z^T X (or X^T X)
  double* ns;        // 5 x m*m: Y0, Y1, Z0, Z1, T of the coupled Newton-Schulz iteration
  float* wf;         // m*m   fp32 matrix the row kernel multiplies by
  double* scal;      // [0] c (scaling), [1..3] residual slots of the Newton-Schulz iterations (it % 3)
  int* nsflag;       // [0] converged (sticky), [1] buffer holding the final Z
};

inline int64_t proj_mm(int m) { return m <= kProjMaxM ? (int64_t)m * m : 0; }

inline bool proj_wide(int m) { return m > kProjMaxM && m <= kWideMaxM; }
// row blocks of the tiled Gram kernel for width m (64 x 64 output tiles: the grid is tiles^2 x row blocks)
inline int wide_row_blocks(int m) {
  const int tiles = (m + 63) / 64;
  const int rb = kWideRowBlocks / (tiles * tiles);
  return rb < 1 ? 1 : rb;
}

inline int64_t proj_ws_doubles(int m) {
  int64_t k = (int64_t)m + proj_mm(m);
  int64_t base = (int64_t)kProjBlocks * k + 2 * m + proj_mm(m) + 8;
  if (proj_wide(m)) {
    const int64_t mm = (int64_t)m * m;
    base += (int64_t)wide_row_blocks(m) * mm / 2 + 1;  // fpart (floats)
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
    w.fpart = (float*)p; p += (int64_t)wide_row_blocks(m) * mm / 2 + 1;
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
// Enqueue de-mean + sqrt(n) * polar factor.  m <= kWideMaxM.  Sets *w.status; nothing on the device reads it (the
// solver's in-graph retractions run on regardless), the host reads it through mde_project_status.
int enqueue_project_standardized(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st);
// Enqueue Z -= (1/n) X (Z^T X).  m <= kWideMaxM.
int enqueue_tangent_standardized(const float* X, float* Z, int64_t n, int m, const ProjWs& w,
                                 const int* active, cudaStream_t st);

// wide rows (mde_project_wide.cu)
int enqueue_project_standardized_wide(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st);
int enqueue_tangent_standardized_wide(const float* X, float* Z, int64_t n, int m, const ProjWs& w,
                                      const int* active, cudaStream_t st);
// column means of a wide matrix into w.mean (mde_project.cu)
int enqueue_colmean_wide(const float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st);

}  // namespace mde
