// mde_project.cu -- constraint projections as fused row kernels.
//
// Reference semantics (cvxgrp/pymde v0.2.1):
//   _Centered.project_onto_constraint      pymde/constraints.py:106-111   Z -= mean(Z, axis 0)
//   _Standardized.project_onto_constraint  pymde/constraints.py:194-195 -> pymde/util.py:129-171
//        de-mean, thin SVD, sqrt(n) U V^T.  Here: the same polar factor through the m x m Gram,
//        sqrt(n) Xc (Xc^T Xc)^(-1/2), eigen-decomposed on device by a one-warp Jacobi sweep
//        (fp64).  No n x m SVD, no extra n x m temporaries.
//   _Standardized.project_onto_tangent_space pymde/constraints.py:186-192  Z -= (1/n) X (Z^T X)
//
// Every projection is: [moments pass: per-block partial column sums + m x m products]
//                      -> [1-block finalize: fixed-order sum, tiny dense algebra]
//                      -> [apply pass over rows].
// Bytes: centered 2 passes x n*m*4 read + n*m*4 write; standardized the same plus m*m.
#include "mde_project.cuh"

using namespace mde;

namespace {

__device__ __forceinline__ bool inactive(const int* active) { return active != nullptr && *active == 0; }

// ---- moments: column sums of X and G[a][b] = sum_r Z[r][a] * X[r][b] --------------------------
// partial layout per block: [m sums][m*m products]
//
// shift (GRAM only, nullable): the retraction passes X itself and gets the sums and products of X - s, s =
// proj_shift(X), stored in shift_out.  Far from the origin, G - n mu mu^T would cancel most of the fp32 digits of G;
// the shifted rows are as small as the spread of the data, and a constant column gives an exactly zero Gram row.
template <int M, bool GRAM>
__global__ void __launch_bounds__(kProjThreads)
moments_small_kernel(const float* __restrict__ Z, const float* __restrict__ X, int64_t n,
                     double* __restrict__ partials, const float* shift, double* shift_out, const int* active) {
  if (inactive(active)) return;
  constexpr int K = GRAM ? (M + M * M) : M;
  float acc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) acc[k] = 0.0f;
  double dacc[K];
#pragma unroll
  for (int k = 0; k < K; ++k) dacc[k] = 0.0;
  float s[M];
#pragma unroll
  for (int c = 0; c < M; ++c) s[c] = 0.0f;
  if (GRAM && shift) {
#pragma unroll
    for (int c = 0; c < M; ++c) s[c] = proj_shift(shift, n, M, c);
    if (blockIdx.x == 0 && threadIdx.x == 0) {
#pragma unroll
      for (int c = 0; c < M; ++c) shift_out[c] = (double)s[c];
    }
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int cnt = 0;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    float x[M], z[M];
#pragma unroll
    for (int c = 0; c < M; ++c) x[c] = X[r * M + c];
    if (GRAM) {
#pragma unroll
      for (int c = 0; c < M; ++c) { x[c] -= s[c]; z[c] = Z[r * M + c] - s[c]; }
    }
#pragma unroll
    for (int c = 0; c < M; ++c) acc[c] += x[c];
    if (GRAM) {
#pragma unroll
      for (int a = 0; a < M; ++a)
#pragma unroll
        for (int b = 0; b < M; ++b) acc[M + a * M + b] += z[a] * x[b];
    }
    if (++cnt == 64) {  // bound fp32 partial length
#pragma unroll
      for (int k = 0; k < K; ++k) { dacc[k] += (double)acc[k]; acc[k] = 0.0f; }
      cnt = 0;
    }
  }
#pragma unroll
  for (int k = 0; k < K; ++k) dacc[k] += (double)acc[k];
  __shared__ double sm[K * 32];
  block_sum<K>(dacc, sm);
  if (threadIdx.x == 0) {
    double* o = partials + (int64_t)blockIdx.x * (M + M * M);
#pragma unroll
    for (int k = 0; k < K; ++k) o[k] = dacc[k];
  }
}

// generic 5 <= m <= 32: one warp per row, lane a owns column a and Gram row a
template <bool GRAM>
__global__ void __launch_bounds__(kProjThreads)
moments_warp_kernel(const float* __restrict__ Z, const float* __restrict__ X, int64_t n, int m,
                    double* __restrict__ partials, const float* shift, double* shift_out, const int* active) {
  if (inactive(active)) return;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float sum = 0.0f;
  float acc[32];
#pragma unroll
  for (int b = 0; b < 32; ++b) acc[b] = 0.0f;
  float s = 0.0f;  // see moments_small_kernel
  if (GRAM && shift && lane < m) {
    s = proj_shift(shift, n, m, lane);
    if (blockIdx.x == 0 && w == 0) shift_out[lane] = (double)s;
  }
  const int64_t stride = (int64_t)gridDim.x * nw;
  for (int64_t r = (int64_t)blockIdx.x * nw + w; r < n; r += stride) {
    float x = (lane < m) ? X[r * m + lane] : 0.0f;
    if (GRAM) x -= s;
    sum += x;
    if (GRAM) {
      float z = (lane < m) ? Z[r * m + lane] - s : 0.0f;
#pragma unroll
      for (int b = 0; b < 32; ++b) {
        float xb = __shfl_sync(kFull, x, b);
        acc[b] += z * xb;
      }
    }
  }
  __shared__ float sm[kProjThreads / 32][33][33];
  sm[w][32][lane] = sum;
  if (GRAM) {
#pragma unroll
    for (int b = 0; b < 32; ++b) sm[w][lane][b] = acc[b];
  }
  __syncthreads();
  double* o = partials + (int64_t)blockIdx.x * (m + m * m);
  const int K = GRAM ? (m + m * m) : m;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    double s = 0.0;
    if (k < m) {
      for (int q = 0; q < nw; ++q) s += (double)sm[q][32][k];
    } else {
      int a = (k - m) / m, b = (k - m) % m;
      for (int q = 0; q < nw; ++q) s += (double)sm[q][a][b];
    }
    o[k] = s;
  }
}

// wide rows (m > 32): column sums only.  thread t owns column t % mpad of row-lane t / mpad.  shift (nullable): sums
// of X - s, s = proj_shift(shift), stored in shift_out (see moments_small_kernel).
__global__ void __launch_bounds__(kProjThreads)
colsum_wide_kernel(const float* __restrict__ X, int64_t n, int m, int mpad,
                   double* __restrict__ partials, const float* shift, double* shift_out, const int* active) {
  if (inactive(active)) return;
  __shared__ double sm[kProjThreads];
  const int nrl = mpad >= kProjThreads ? 1 : kProjThreads / mpad;
  const int rl = threadIdx.x / mpad, c0 = threadIdx.x % mpad;
  for (int cb = 0; cb < m; cb += kProjThreads) {  // column blocks of 256 (m > 256 only loops)
    int c = cb + c0;
    double acc = 0.0;
    if (c < m && rl < nrl) {
      float s = 0.0f;
      if (shift) {
        s = proj_shift(shift, n, m, c);
        if (blockIdx.x == 0 && rl == 0) shift_out[c] = (double)s;
      }
      float facc = 0.0f;
      int cnt = 0;
      for (int64_t r = (int64_t)blockIdx.x * nrl + rl; r < n; r += (int64_t)gridDim.x * nrl) {
        facc += shift ? X[r * m + c] - s : X[r * m + c];
        if (++cnt == 64) { acc += (double)facc; facc = 0.0f; cnt = 0; }
      }
      acc += (double)facc;
    }
    sm[threadIdx.x] = acc;
    __syncthreads();
    if (rl == 0 && c < m) {
      double s = 0.0;
      for (int q = 0; q < nrl; ++q) s += sm[q * mpad + c0];
      partials[(int64_t)blockIdx.x * m + c] = s;
    }
    __syncthreads();
  }
}

__global__ void colmean_finalize_kernel(const double* __restrict__ partials, int nblocks, int64_t n, int m,
                                        const double* shift, double* __restrict__ mean, const int* active) {
  if (inactive(active)) return;
  // one warp per column
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int k = gw; k < m; k += nw) {
    double s = 0.0;
    for (int b = lane; b < nblocks; b += 32) s += partials[(int64_t)b * m + k];
    s = warp_sum(s);
    if (lane == 0) mean[k] = shift ? shift[k] + s / (double)n : s / (double)n;
  }
}

// ---- one-warp cyclic Jacobi on a symmetric m x m matrix in shared memory (fp64) -----------
// On exit A's diagonal holds the eigenvalues, V the eigenvectors (columns).
__device__ void jacobi_eig_warp(double* A, double* V, int m) {
  const int lane = threadIdx.x & 31;
  for (int i = lane; i < m * m; i += 32) V[i] = ((i / m) == (i % m)) ? 1.0 : 0.0;
  __syncwarp();
  for (int sweep = 0; sweep < 30; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int i = lane; i < m * m; i += 32) {
      double v = A[i];
      if ((i / m) == (i % m)) diag += v * v; else off += v * v;
    }
    off = warp_sum(off); diag = warp_sum(diag);
    if (off <= 1e-30 * diag || off == 0.0) break;
    for (int p = 0; p < m - 1; ++p) {
      for (int q = p + 1; q < m; ++q) {
        double apq = A[p * m + q];
        if (fabs(apq) > 1e-300) {
          double app = A[p * m + p], aqq = A[q * m + q];
          double theta = (aqq - app) / (2.0 * apq);
          double t = (theta >= 0.0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
          __syncwarp();
          // columns p, q of A and V
          if (lane < m) {
            int k = lane;
            double akp = A[k * m + p], akq = A[k * m + q];
            A[k * m + p] = c * akp - s * akq;
            A[k * m + q] = s * akp + c * akq;
            double vkp = V[k * m + p], vkq = V[k * m + q];
            V[k * m + p] = c * vkp - s * vkq;
            V[k * m + q] = s * vkp + c * vkq;
          }
          __syncwarp();
          // rows p, q of A
          if (lane < m) {
            int k = lane;
            double apk = A[p * m + k], aqk = A[q * m + k];
            A[p * m + k] = c * apk - s * aqk;
            A[q * m + k] = s * apk + c * aqk;
          }
          __syncwarp();
        }
      }
    }
  }
  __syncwarp();
}

// MODE 0: mean only.  MODE 1: the partials are moments of X - s (s = shift), d = mean(X - s):
// mean = s + d and W = sqrt(n) (Gc)^(-1/2), Gc = G_s - n d d^T.  MODE 2: mat = G / n (tangent).
template <int MODE>
__global__ void __launch_bounds__(256)
proj_finalize_kernel(const double* __restrict__ partials, int nblocks, int64_t n, int m,
                     double* __restrict__ mean, const double* __restrict__ shift, double* __restrict__ mat,
                     int* status, const int* active) {
  if (inactive(active)) return;
  __shared__ double sA[kProjMaxM * kProjMaxM];
  __shared__ double sV[kProjMaxM * kProjMaxM];
  __shared__ double sMu[kProjMaxM];
  const int K = m + m * m;
  const int Kuse = (MODE == 0) ? m : K;
  // fixed-order reduction over blocks: one WARP per output (lanes stride the blocks, then a
  // shuffle tree) -- deterministic for a given launch shape, and ~nblocks/32 dependent loads deep
  {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
    for (int k = w; k < Kuse; k += nw) {
      double s = 0.0;
      for (int b = lane; b < nblocks; b += 32) s += partials[(int64_t)b * K + k];
      s = warp_sum(s);
      if (lane == 0) {
        if (k < m) sMu[k] = s / (double)n;
        else sA[k - m] = s;
      }
    }
  }
  __syncthreads();
  if (MODE == 0) {
    for (int k = threadIdx.x; k < m; k += blockDim.x) mean[k] = sMu[k];
  }
  if (MODE == 1) {
    for (int k = threadIdx.x; k < m; k += blockDim.x) mean[k] = shift[k] + sMu[k];
  }
  if (MODE == 0) return;
  if (MODE == 2) {
    for (int k = threadIdx.x; k < m * m; k += blockDim.x) mat[k] = sA[k] / (double)n;
    return;
  }
  // MODE 1
  for (int k = threadIdx.x; k < m * m; k += blockDim.x) {
    int a = k / m, b = k % m;
    sA[k] -= (double)n * sMu[a] * sMu[b];
  }
  __syncthreads();
  // symmetrise (rounding) then eigen-decompose on warp 0
  if (threadIdx.x < 32) {
    for (int k = threadIdx.x; k < m * m; k += 32) {
      int a = k / m, b = k % m;
      if (a < b) { double v = 0.5 * (sA[a * m + b] + sA[b * m + a]); sA[a * m + b] = v; sA[b * m + a] = v; }
    }
    __syncwarp();
    jacobi_eig_warp(sA, sV, m);
    // The de-meaned X has rank <= n - 1.  A Gram that is singular in exact arithmetic keeps eigenvalues of the
    // order of its rounding, of either sign: the test is relative to the largest.
    bool bad = n <= (int64_t)m;
    double lmin = sA[0], lmax = sA[0];
    for (int k = 0; k < m; ++k) {
      const double l = sA[k * m + k];
      if (!isfinite(l)) bad = true;
      lmin = fmin(lmin, l); lmax = fmax(lmax, l);
    }
    if (!(lmin > kProjRankTol * lmax)) bad = true;
    if (threadIdx.x == 0 && status) *status = bad ? 1 : 0;
    const double sq = sqrt((double)n);
    for (int k = threadIdx.x; k < m * m; k += 32) {
      int a = k / m, b = k % m;
      double s = 0.0;
      for (int e = 0; e < m; ++e) s += sV[a * m + e] * sV[b * m + e] / sqrt(sA[e * m + e]);
      mat[k] = sq * s;
    }
  }
}

// ---- apply passes ------------------------------------------------------------------------
__global__ void __launch_bounds__(kProjThreads)
center_apply_kernel(float* __restrict__ X, int64_t total, int m, const double* __restrict__ mean,
                    const int* active) {
  if (inactive(active)) return;
  extern __shared__ float smu[];
  for (int c = threadIdx.x; c < m; c += blockDim.x) smu[c] = (float)mean[c];
  __syncthreads();
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride)
    X[i] -= smu[i % m];
}

// MODE 0: X <- (X - mu) W          (retraction, in place)
// MODE 1: Z <- Z - X Mat           (tangent projection, in place on Z)
template <int M, int MODE>
__global__ void __launch_bounds__(kProjThreads)
rowmat_small_kernel(const float* __restrict__ X, float* __restrict__ Y, int64_t n,
                    const double* __restrict__ mean, const double* __restrict__ mat, const int* active) {
  if (inactive(active)) return;
  float W[M * M], mu[M];
#pragma unroll
  for (int k = 0; k < M * M; ++k) W[k] = (float)mat[k];
#pragma unroll
  for (int k = 0; k < M; ++k) mu[k] = (MODE == 0) ? (float)mean[k] : 0.0f;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += stride) {
    float x[M], o[M];
#pragma unroll
    for (int c = 0; c < M; ++c) x[c] = X[r * M + c] - mu[c];
#pragma unroll
    for (int b = 0; b < M; ++b) {
      float s = 0.0f;
#pragma unroll
      for (int a = 0; a < M; ++a) s += x[a] * W[a * M + b];
      o[b] = s;
    }
    if (MODE == 0) {
#pragma unroll
      for (int c = 0; c < M; ++c) Y[r * M + c] = o[c];
    } else {
#pragma unroll
      for (int c = 0; c < M; ++c) Y[r * M + c] -= o[c];
    }
  }
}

template <int MODE>
__global__ void __launch_bounds__(kProjThreads)
rowmat_warp_kernel(const float* __restrict__ X, float* __restrict__ Y, int64_t n, int m,
                   const double* __restrict__ mean, const double* __restrict__ mat, const int* active) {
  if (inactive(active)) return;
  __shared__ float sW[kProjMaxM * kProjMaxM];
  __shared__ float sMu[kProjMaxM];
  for (int k = threadIdx.x; k < m * m; k += blockDim.x) sW[k] = (float)mat[k];
  for (int k = threadIdx.x; k < m; k += blockDim.x) sMu[k] = (MODE == 0) ? (float)mean[k] : 0.0f;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int64_t stride = (int64_t)gridDim.x * nw;
  for (int64_t r = (int64_t)blockIdx.x * nw + w; r < n; r += stride) {
    float x = (lane < m) ? X[r * m + lane] - sMu[lane] : 0.0f;
    float s = 0.0f;
    for (int a = 0; a < m; ++a) {
      float xa = __shfl_sync(kFull, x, a);
      if (lane < m) s += xa * sW[a * m + lane];
    }
    if (lane < m) {
      if (MODE == 0) Y[r * m + lane] = s;
      else Y[r * m + lane] -= s;
    }
  }
}

int blocks_for_rows(int64_t n, int rows_per_block) {
  int64_t nb = (n + rows_per_block - 1) / rows_per_block;
  if (nb < 1) nb = 1;
  if (nb > kProjBlocks) nb = kProjBlocks;
  return (int)nb;
}

// shift: null, or the row (X[0]) the retraction's Gram is taken around (see moments_small_kernel)
template <bool GRAM>
int launch_moments(const float* Z, const float* X, int64_t n, int m, const float* shift, const ProjWs& w,
                   const int* active, int* nblocks, cudaStream_t st) {
  int nb;
  double* so = w.shift;
  if (m <= 4) {
    nb = blocks_for_rows(n, kProjThreads);
    switch (m) {
      case 1: moments_small_kernel<1, GRAM><<<nb, kProjThreads, 0, st>>>(Z, X, n, w.partials, shift, so, active); break;
      case 2: moments_small_kernel<2, GRAM><<<nb, kProjThreads, 0, st>>>(Z, X, n, w.partials, shift, so, active); break;
      case 3: moments_small_kernel<3, GRAM><<<nb, kProjThreads, 0, st>>>(Z, X, n, w.partials, shift, so, active); break;
      default: moments_small_kernel<4, GRAM><<<nb, kProjThreads, 0, st>>>(Z, X, n, w.partials, shift, so, active); break;
    }
  } else {
    nb = blocks_for_rows(n, kProjThreads / 32);
    moments_warp_kernel<GRAM><<<nb, kProjThreads, 0, st>>>(Z, X, n, m, w.partials, shift, so, active);
  }
  MDE_LAUNCH_CHECK();
  *nblocks = nb;
  return 0;
}

template <int MODE>
int launch_rowmat(const float* X, float* Y, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st) {
  if (m <= 4) {
    int nb = blocks_for_rows(n, kProjThreads);
    switch (m) {
      case 1: rowmat_small_kernel<1, MODE><<<nb, kProjThreads, 0, st>>>(X, Y, n, w.mean, w.mat, active); break;
      case 2: rowmat_small_kernel<2, MODE><<<nb, kProjThreads, 0, st>>>(X, Y, n, w.mean, w.mat, active); break;
      case 3: rowmat_small_kernel<3, MODE><<<nb, kProjThreads, 0, st>>>(X, Y, n, w.mean, w.mat, active); break;
      default: rowmat_small_kernel<4, MODE><<<nb, kProjThreads, 0, st>>>(X, Y, n, w.mean, w.mat, active); break;
    }
  } else {
    int nb = blocks_for_rows(n, kProjThreads / 32);
    rowmat_warp_kernel<MODE><<<nb, kProjThreads, 0, st>>>(X, Y, n, m, w.mean, w.mat, active);
  }
  MDE_LAUNCH_CHECK();
  return 0;
}

}  // namespace

namespace mde {

int enqueue_colmean_wide(const float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st,
                         const float* shift) {
  int mpad = 64;
  while (mpad < m && mpad < kProjThreads) mpad <<= 1;
  int nrl = kProjThreads / mpad;
  const int nb = blocks_for_rows(n, nrl * 8);
  colsum_wide_kernel<<<nb, kProjThreads, 0, st>>>(X, n, m, mpad, w.partials, shift, w.shift, active);
  MDE_LAUNCH_CHECK();
  colmean_finalize_kernel<<<(m + 7) / 8, 256, 0, st>>>(w.partials, nb, n, m, shift ? w.shift : nullptr, w.mean, active);
  MDE_LAUNCH_CHECK();
  return 0;
}

int enqueue_project_centered(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st) {
  int nb = 0, rc;
  if (m <= kProjMaxM) {
    if ((rc = launch_moments<false>(X, X, n, m, nullptr, w, active, &nb, st))) return rc;
    proj_finalize_kernel<0><<<1, 256, 0, st>>>(w.partials, nb, n, m, w.mean, w.shift, w.mat, w.status, active);
    MDE_LAUNCH_CHECK();
  } else if ((rc = enqueue_colmean_wide(X, n, m, w, active, st))) return rc;
  int64_t total = n * m;
  int nbb = (int)((total + kProjThreads * 4 - 1) / (kProjThreads * 4));
  if (nbb > kProjBlocks * 4) nbb = kProjBlocks * 4;
  if (nbb < 1) nbb = 1;
  center_apply_kernel<<<nbb, kProjThreads, m * sizeof(float), st>>>(X, total, m, w.mean, active);
  MDE_LAUNCH_CHECK();
  return 0;
}

int enqueue_project_standardized(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st) {
  if (proj_wide(m)) return enqueue_project_standardized_wide(X, n, m, w, active, st);
  if (m > kProjMaxM) return MDE_E_UNSUPPORTED;
  int nb = 0, rc;
  if ((rc = launch_moments<true>(X, X, n, m, X, w, active, &nb, st))) return rc;
  proj_finalize_kernel<1><<<1, 256, 0, st>>>(w.partials, nb, n, m, w.mean, w.shift, w.mat, w.status, active);
  MDE_LAUNCH_CHECK();
  return launch_rowmat<0>(X, X, n, m, w, active, st);
}

int enqueue_tangent_standardized(const float* X, float* Z, int64_t n, int m, const ProjWs& w,
                                 const int* active, cudaStream_t st) {
  if (proj_wide(m)) return enqueue_tangent_standardized_wide(X, Z, n, m, w, active, st);
  if (m > kProjMaxM) return MDE_E_UNSUPPORTED;
  int nb = 0, rc;
  if ((rc = launch_moments<true>(Z, X, n, m, nullptr, w, active, &nb, st))) return rc;
  proj_finalize_kernel<2><<<1, 256, 0, st>>>(w.partials, nb, n, m, w.mean, w.shift, w.mat, w.status, active);
  MDE_LAUNCH_CHECK();
  return launch_rowmat<1>(X, Z, n, m, w, active, st);
}

}  // namespace mde

extern "C" {

int64_t mde_project_ws_bytes(int64_t n, int m) {
  (void)n;
  return (int64_t)sizeof(double) * proj_ws_doubles(m) + 64;
}

int mde_project_centered(float* X, int64_t n, int m, void* ws, void* stream) {
  if (!X || !ws || n < 1 || m < 1) return MDE_E_INVALID;
  return enqueue_project_centered(X, n, m, proj_ws_carve(ws, m), nullptr, (cudaStream_t)stream);
}

int mde_project_standardized(float* X, int64_t n, int m, void* ws, void* stream) {
  if (!X || !ws || n < 1 || m < 1) return MDE_E_INVALID;
  if (m > kWideMaxM) return MDE_E_UNSUPPORTED;
  return enqueue_project_standardized(X, n, m, proj_ws_carve(ws, m), nullptr, (cudaStream_t)stream);
}

int mde_project_status(const void* ws, int m, int* status, void* stream) {
  if (!ws || !status || m < 1) return MDE_E_INVALID;
  const ProjWs w = proj_ws_carve(const_cast<void*>(ws), m);
  const cudaStream_t st = (cudaStream_t)stream;
  MDE_CUDA_TRY(cudaMemcpyAsync(status, w.status, sizeof(int), cudaMemcpyDeviceToHost, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

int mde_tangent_standardized(const float* X, float* Z, int64_t n, int m, void* ws, void* stream) {
  if (!X || !Z || !ws || n < 1 || m < 1) return MDE_E_INVALID;
  if (m > kWideMaxM) return MDE_E_UNSUPPORTED;
  return enqueue_tangent_standardized(X, Z, n, m, proj_ws_carve(ws, m), nullptr, (cudaStream_t)stream);
}

}  // extern "C"
