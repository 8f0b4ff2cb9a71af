// mde_project_wide.cu -- the Standardized constraint for wide embeddings, 32 < m <= 1024, on the device.
//
// Reference: pymde/constraints.py:167-200 -> pymde/util.py:129-171 (de-mean, thin SVD of the n x m matrix,
// sqrt(n) U V^T; pinned at m = 250 by pymde/test_util.py:20-71) and pymde/constraints.py:186-192 (tangent space:
// Z -= (1/n) X (Z^T X)).  The narrow path (mde_project.cu) eigen-decomposes the m x m Gram matrix in one warp; that
// does not scale to m = 256.  Here everything is a tiled product:
//
//   gram      P[rb] = Z[rows rb]^T X[rows rb]   64 x 64 output tiles, 4 x 4 per thread (m <= 256), or 128 x 128, 8 x 8
//                                               per thread (m > 256); fp32 inside a row block of <= ceil(n / 16) rows
//   reduce    G = sum_rb P[rb]                  fp64 across row blocks (fixed order)
//   retraction:   G is the Gram of X - s (s = proj_shift, near the column mean) ;  A = (G - n (mu - s)(mu - s)^T) / n ;
//                 W = A^(-1/2) by the coupled Newton-Schulz iteration
//                     Y_0 = A / c, Z_0 = I ;  T = (3 I - Z Y) / 2 ;  Y <- Y T ;  Z <- T Z      (Z -> sqrt(c) A^(-1/2))
//                 in fp64 with c = ||A||_inf >= lambda_max (so the iteration converges for every positive definite
//                 A); an embedding that is already nearly standardized -- every trial point of the solver -- has
//                 A = I + E and needs 4-6 iterations.  The iterations are enqueued as a FIXED chain (CUDA-graph
//                 capturable) and switch themselves off through a device flag once ||I - Z Y||_F < 1e-9 m.  The
//                 m x m products run on FFMA up to m = 256 and on the fp64 tensor cores (DMMA) above.
//   rowmat    X <- (X - mu) W   or   Z <- Z - X (G / n).  m <= 256: 32 rows x all columns per block, the block's rows
//             held in shared memory (which makes the in-place update safe), the matrix streamed in 16-row slabs.
//             m > 256: 128 x 128 output tiles like the Gram; the retraction writes each chunk of 16 m rows to the
//             (then free) fpart region and copies it back.
//
// Every kernel takes the solver's `active` gate like the narrow path.
#include "mde_project.cuh"

using namespace mde;

namespace {

__device__ __forceinline__ bool inactive(const int* active) { return active != nullptr && *active == 0; }

constexpr int kGK = 16;   // rows per shared-memory stage

// P[rb][a][b] = sum over the rows of row block rb of (Z[r][a] - s[a]) (X[r][b] - s[b]);  grid = (tiles*tiles, row
// blocks), T = 16 TM output tiles, TM x TM per thread.  s = proj_shift(shift) (nullable; the retraction passes X, and
// s goes to shift_out): the products of the shifted rows keep the fp32 digits that G - n mu mu^T would cancel when the
// columns sit far from the origin.  A thread owns rows (and columns) t * 4 + (i & 3) + 64 (i >> 2), i < TM, of the
// tile; each of its sums runs over the block's rows in order, so the tile size does not change any P element.
template <int TM>
__global__ void __launch_bounds__(256, TM == 8 ? 2 : 0)
gram_wide_kernel(const float* __restrict__ Z, const float* __restrict__ X, int64_t n, int m, int tiles,
                 int64_t rows_per_block, float* __restrict__ P, const float* shift, double* shift_out,
                 const int* active) {
  constexpr int T = 16 * TM;
  constexpr int Q = kGK * T / 256;  // staged elements per thread and operand
  if (inactive(active)) return;
  __shared__ __align__(16) float sA[kGK][T + 4];
  __shared__ __align__(16) float sB[kGK][T + 4];
  const int ta = blockIdx.x / tiles, tb = blockIdx.x % tiles;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  // every element this thread stages lies in column threadIdx.x % T of the two tiles
  float sa = 0.0f, sb = 0.0f;
  if (shift) {
    const int ca = ta * T + (threadIdx.x % T), cb = tb * T + (threadIdx.x % T);
    if (ca < m) sa = proj_shift(shift, n, m, ca);
    if (cb < m) sb = proj_shift(shift, n, m, cb);
    if (blockIdx.y == 0 && tb == 0 && threadIdx.x < T && ca < m) shift_out[ca] = (double)sa;
  }
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_block;
  int64_t r1 = r0 + rows_per_block;
  if (r1 > n) r1 = n;
  float acc[TM][TM];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TM; ++j) acc[i][j] = 0.0f;
  for (int64_t r = r0; r < r1; r += kGK) {
    // kGK rows x T columns of each operand
#pragma unroll
    for (int q = 0; q < Q; ++q) {
      const int e = threadIdx.x + 256 * q;
      const int kk = e / T, c = e % T;
      const int64_t row = r + kk;
      const int ca = ta * T + c, cb = tb * T + c;
      sA[kk][c] = (row < r1 && ca < m) ? Z[row * m + ca] - sa : 0.0f;
      sB[kk][c] = (row < r1 && cb < m) ? X[row * m + cb] - sb : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGK; ++kk) {
      float a[TM], b[TM];
#pragma unroll
      for (int h = 0; h < TM / 4; ++h) {
        const float4 av = *reinterpret_cast<const float4*>(&sA[kk][ty * 4 + 64 * h]);
        const float4 bv = *reinterpret_cast<const float4*>(&sB[kk][tx * 4 + 64 * h]);
        a[4 * h] = av.x; a[4 * h + 1] = av.y; a[4 * h + 2] = av.z; a[4 * h + 3] = av.w;
        b[4 * h] = bv.x; b[4 * h + 1] = bv.y; b[4 * h + 2] = bv.z; b[4 * h + 3] = bv.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TM; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* out = P + (int64_t)blockIdx.y * m * m;
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int a = ta * T + ty * 4 + (i & 3) + 64 * (i >> 2);
#pragma unroll
    for (int j = 0; j < TM; ++j) {
      const int b = tb * T + tx * 4 + (j & 3) + 64 * (j >> 2);
      if (a < m && b < m) out[(int64_t)a * m + b] = acc[i][j];
    }
  }
}

// G[k] = sum_rb P[rb][k]  (fp64, fixed order)
__global__ void __launch_bounds__(256)
gram_reduce_kernel(const float* __restrict__ P, int row_blocks, int64_t mm, double* __restrict__ G, const int* active) {
  if (inactive(active)) return;
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= mm) return;
  double s0 = 0.0, s1 = 0.0;
  int rb = 0;
  for (; rb + 1 < row_blocks; rb += 2) { s0 += (double)P[(int64_t)rb * mm + k]; s1 += (double)P[(int64_t)(rb + 1) * mm + k]; }
  if (rb < row_blocks) s0 += (double)P[(int64_t)rb * mm + k];
  G[k] = s0 + s1;
}

// tangent: wf = G / n (fp32 matrix of the row kernel)
__global__ void __launch_bounds__(256)
tangent_mat_kernel(const double* __restrict__ G, int64_t mm, double inv_n, float* __restrict__ wf, const int* active) {
  if (inactive(active)) return;
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < mm) wf[k] = (float)(G[k] * inv_n);
}

// retraction: A = sym(G_s - n d d^T) / n with d = mu - s (G_s is the Gram of X - s), c = ||A||_inf, Y0 = A / c,
// Z0 = I, flags cleared.  One block.
__global__ void __launch_bounds__(1024)
ns_init_kernel(const double* __restrict__ G, const double* __restrict__ mean, const double* __restrict__ shift,
               int64_t n, int m, double* __restrict__ Y0, double* __restrict__ Z0, double* __restrict__ scal,
               int* __restrict__ nsflag, int* status, const int* active) {
  if (inactive(active)) return;
  __shared__ double s_row[kWideMaxM];
  __shared__ double s_d[kWideMaxM];
  __shared__ double s_c;
  const double dn = (double)n;
  for (int a = threadIdx.x; a < m; a += blockDim.x) s_d[a] = mean[a] - shift[a];
  __syncthreads();
  for (int a = threadIdx.x; a < m; a += blockDim.x) {
    double rs = 0.0;
    for (int b = 0; b < m; ++b) {
      const double v = 0.5 * (G[(int64_t)a * m + b] + G[(int64_t)b * m + a]) - dn * s_d[a] * s_d[b];
      rs += fabs(v);
    }
    s_row[a] = rs / dn;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0;
    bool bad = n <= (int64_t)m;  // the de-meaned X has rank <= n - 1
    for (int a = 0; a < m; ++a) { c = fmax(c, s_row[a]); if (!isfinite(s_row[a])) bad = true; }
    if (!(c > 0.0)) { bad = true; c = 1.0; }
    s_c = c;
    scal[0] = c; scal[1] = 0.0; scal[2] = 0.0; scal[3] = 0.0;
    nsflag[0] = 0; nsflag[1] = 0;
    if (status) *status = bad ? 1 : 0;
  }
  __syncthreads();
  const double ic = 1.0 / (s_c * dn);
  for (int k = threadIdx.x; k < m * m; k += blockDim.x) {
    const int a = k / m, b = k % m;
    Y0[k] = (0.5 * (G[(int64_t)a * m + b] + G[(int64_t)b * m + a]) - dn * s_d[a] * s_d[b]) * ic;
    Z0[k] = (a == b) ? 1.0 : 0.0;
  }
}

// C = alpha A B + beta I on m x m fp64 matrices.  blockIdx.z selects one of two independent products (Y T and T Z in
// one launch).
//
// Gating of the fixed chain: iteration `it` accumulates r_it = ||I - Z_it Y_it||_F^2 into slot it % 3 (first kernel,
// RES).  A kernel of iteration it idles when the sticky flag is set (by an EARLIER launch) or when r_(it-1) < tol^2;
// both are stable while the kernel runs, so all its blocks decide alike.  The first kernel that sees r_(it-1) < tol^2
// sets the flag and records which buffer holds the final Z (the update of iteration it - 1 was still applied: it only
// improves the iterate).  The second kernel of an iteration zeroes the slot of the next one.
struct MmArgs { const double* A; const double* B; double* C; };

// true: this launch of the chain idles
template <bool RES>
__device__ __forceinline__ bool ns_gate(const double* res_prev, double* res_zero, double tol2, int* nsflag, int cur) {
  const bool first = blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && threadIdx.x == 0;
  if (nsflag[0]) return true;
  if (res_prev != nullptr && *res_prev < tol2) {
    if (RES && first) { nsflag[1] = cur; __threadfence(); nsflag[0] = 1; }
    return true;
  }
  if (!RES && first && res_zero) *res_zero = 0.0;
  return false;
}

// m <= 256: 32 x 32 tiles, 2 x 2 per thread on FFMA
template <bool RES>
__global__ void __launch_bounds__(256)
ns_mm_kernel(MmArgs p0, MmArgs p1, int m, double alpha, double beta, double* __restrict__ res_acc,
             const double* __restrict__ res_prev, double* __restrict__ res_zero, double tol2, int* __restrict__ nsflag,
             int cur, const int* active) {
  if (inactive(active)) return;
  if (ns_gate<RES>(res_prev, res_zero, tol2, nsflag, cur)) return;
  const MmArgs p = blockIdx.z ? p1 : p0;
  __shared__ double sA[32][17];
  __shared__ double sB[16][33];
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  const int a0 = blockIdx.y * 32, b0 = blockIdx.x * 32;
  double acc[2][2] = {{0.0, 0.0}, {0.0, 0.0}};
  for (int k0 = 0; k0 < m; k0 += 16) {
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int e = threadIdx.x + 256 * q;
      { const int r = e >> 4, c = e & 15; const int a = a0 + r, k = k0 + c; sA[r][c] = (a < m && k < m) ? p.A[(int64_t)a * m + k] : 0.0; }
      { const int r = e >> 5, c = e & 31; const int k = k0 + r, b = b0 + c; sB[r][c] = (k < m && b < m) ? p.B[(int64_t)k * m + b] : 0.0; }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      const double x0 = sA[ty * 2][kk], x1 = sA[ty * 2 + 1][kk];
      const double y0 = sB[kk][tx * 2], y1 = sB[kk][tx * 2 + 1];
      acc[0][0] = fma(x0, y0, acc[0][0]); acc[0][1] = fma(x0, y1, acc[0][1]);
      acc[1][0] = fma(x1, y0, acc[1][0]); acc[1][1] = fma(x1, y1, acc[1][1]);
    }
    __syncthreads();
  }
  double r2 = 0.0;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int a = a0 + ty * 2 + i, b = b0 + tx * 2 + j;
      if (a < m && b < m) {
        const double id = (a == b) ? 1.0 : 0.0;
        if (RES) { const double e = id - acc[i][j]; r2 += e * e; }
        p.C[(int64_t)a * m + b] = alpha * acc[i][j] + beta * id;
      }
    }
  if (RES) {
    r2 = warp_sum(r2);
    if ((threadIdx.x & 31) == 0 && r2 != 0.0) atomicAdd(res_acc, r2);
  }
}

// m > 256: 64 x 64 tiles on the fp64 tensor cores, mma.m16n8k16 (DMMA.16x8x16); 4 warps of 32 x 32, k staged 32 at
// a time.  Fragments (g = lane / 4, t = lane % 4): A a_q at (g + 8 (q & 1), t + 4 (q >> 1)), B b_q at (t + 4 q, g),
// C c_q at (g + 8 (q >> 1), 2 t + (q & 1)).  Each element is an fp64 sum of the same products as the FFMA kernel's.
constexpr int kDT = 64, kDK = 32;
__device__ __forceinline__ void dmma16816(double (&d)[4], const double (&a)[8], const double (&b)[4]) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, "
               "{%12,%13,%14,%15}, {%0,%1,%2,%3};"
               : "+d"(d[0]), "+d"(d[1]), "+d"(d[2]), "+d"(d[3])
               : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]),
                 "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
}

template <bool RES>
__global__ void __launch_bounds__(128)
ns_dmma_kernel(MmArgs p0, MmArgs p1, int m, double alpha, double beta, double* __restrict__ res_acc,
               const double* __restrict__ res_prev, double* __restrict__ res_zero, double tol2,
               int* __restrict__ nsflag, int cur, const int* active) {
  if (inactive(active)) return;
  if (ns_gate<RES>(res_prev, res_zero, tol2, nsflag, cur)) return;
  const MmArgs p = blockIdx.z ? p1 : p0;
  __shared__ double sA[kDT][kDK + 4];   // A[a0 + r][k0 + c]
  __shared__ double sB[kDK][kDT + 4];   // B[k0 + r][b0 + c]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const int wr = (warp >> 1) * 32, wc = (warp & 1) * 32;
  const int a0 = blockIdx.y * kDT, b0 = blockIdx.x * kDT;
  double acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[i][j][q] = 0.0;
  for (int k0 = 0; k0 < m; k0 += kDK) {
#pragma unroll
    for (int q = 0; q < kDT * kDK / 128; ++q) {
      const int e = threadIdx.x + 128 * q;
      { const int r = e / kDK, c = e % kDK; const int a = a0 + r, k = k0 + c; sA[r][c] = (a < m && k < m) ? p.A[(int64_t)a * m + k] : 0.0; }
      { const int r = e / kDT, c = e % kDT; const int k = k0 + r, b = b0 + c; sB[r][c] = (k < m && b < m) ? p.B[(int64_t)k * m + b] : 0.0; }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kDK; kk += 16) {
      double af[2][8], bf[4][4];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int q = 0; q < 8; ++q) af[i][q] = sA[wr + 16 * i + g + 8 * (q & 1)][kk + t + 4 * (q >> 1)];
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) bf[j][q] = sB[kk + t + 4 * q][wc + 8 * j + g];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) dmma16816(acc[i][j], af[i], bf[j]);
    }
    __syncthreads();
  }
  double r2 = 0.0;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int a = a0 + wr + 16 * i + g + 8 * (q >> 1), b = b0 + wc + 8 * j + 2 * t + (q & 1);
        if (a < m && b < m) {
          const double id = (a == b) ? 1.0 : 0.0;
          if (RES) { const double e = id - acc[i][j][q]; r2 += e * e; }
          p.C[(int64_t)a * m + b] = alpha * acc[i][j][q] + beta * id;
        }
      }
  if (RES) {
    r2 = warp_sum(r2);
    if (lane == 0 && r2 != 0.0) atomicAdd(res_acc, r2);
  }
}

// W = Z_final / sqrt(c) as fp32; status = 1 when the chain ended without converging
__global__ void __launch_bounds__(256)
ns_finish_kernel(const double* __restrict__ ns, int64_t mm, const double* __restrict__ scal, const int* __restrict__ nsflag,
                 int last_buf, const double* __restrict__ res_last, double tol2, float* __restrict__ wf, int* status,
                 const int* active) {
  if (inactive(active)) return;
  const int buf = nsflag[0] ? nsflag[1] : last_buf;
  const double* Zf = ns + (int64_t)(2 + buf) * mm;
  const double s = 1.0 / sqrt(scal[0]);
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k < mm) wf[k] = (float)(Zf[k] * s);
  if (k == 0 && status && !nsflag[0] && !(*res_last < tol2)) *status = 1;
}

// MODE 0: Y[r] = (X[r] - mu) W   (in place allowed: the block's rows are in shared memory before anything is written)
// MODE 1: Y[r] -= X[r] W
template <int MODE>
__global__ void __launch_bounds__(256)
rowmat_wide_kernel(const float* __restrict__ X, float* __restrict__ Y, int64_t n, int m, int mp,
                   const double* __restrict__ mean, const float* __restrict__ W, const int* active) {
  if (inactive(active)) return;
  extern __shared__ float smem[];
  float* sX = smem;                 // [32][mp + 1]
  float* sW = smem + 32 * (mp + 1); // [16][mp]
  const int ty = threadIdx.x >> 5, tx = threadIdx.x & 31;
  const int64_t tiles = (n + 31) / 32;
  for (int64_t t = blockIdx.x; t < tiles; t += gridDim.x) {
    const int64_t r0 = t * 32;
    __syncthreads();  // previous tile's sX / sW readers are done
    for (int e = threadIdx.x; e < 32 * m; e += 256) {
      const int rr = e / m, c = e % m;
      const int64_t row = r0 + rr;
      float v = (row < n) ? X[row * m + c] : 0.0f;
      if (MODE == 0) v -= (float)mean[c];
      sX[rr * (mp + 1) + c] = v;
    }
    float acc[4][8];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
    for (int k0 = 0; k0 < m; k0 += 16) {
      __syncthreads();
      for (int e = threadIdx.x; e < 16 * mp; e += 256) {
        const int kk = e / mp, c = e % mp;
        sW[e] = (k0 + kk < m && c < m) ? W[(int64_t)(k0 + kk) * m + c] : 0.0f;
      }
      __syncthreads();
      const int kmax = (m - k0 < 16) ? m - k0 : 16;
      for (int kk = 0; kk < kmax; ++kk) {
        float x[4], w[8];
#pragma unroll
        for (int i = 0; i < 4; ++i) x[i] = sX[(ty * 4 + i) * (mp + 1) + k0 + kk];
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = (tx + 32 * j < mp) ? sW[kk * mp + tx + 32 * j] : 0.0f;
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(x[i], w[j], acc[i][j]);
      }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t row = r0 + ty * 4 + i;
      if (row >= n) continue;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int c = tx + 32 * j;
        if (c < m) {
          if (MODE == 0) Y[row * m + c] = acc[i][j];
          else Y[row * m + c] -= acc[i][j];
        }
      }
    }
  }
}

// m > 256: O = (X - mu) W  (MODE 0)  or  O = B - X W  (MODE 1) over `rows` rows, as 128 x 128 output tiles, 8 x 8 per
// thread, k staged kGK at a time -- the Gram kernel's layout with X as the row operand.  O may be B (the tangent: Z is
// not read by the product) but not X: the retraction writes its rows to a staging region and copies them back.  Each
// output is the ascending fp32 sum over k, as in rowmat_wide_kernel.
template <int MODE>
__global__ void __launch_bounds__(256, 2)
rowgemm_kernel(const float* __restrict__ X, const float* B, float* O, int rows, int m,
               const double* __restrict__ mean, const float* __restrict__ W, const int* active) {
  constexpr int T = 128;
  if (inactive(active)) return;
  __shared__ __align__(16) float sA[kGK][T + 4];  // sA[k][r] = X[r0 + r][k0 + k] (- mu)
  __shared__ __align__(16) float sB[kGK][T + 4];  // sB[k][c] = W[k0 + k][c0 + c]
  const int r0 = blockIdx.y * T;  // rows * m < 2^31: a chunk is at most the fpart region
  const int c0 = blockIdx.x * T;
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.0f;
  for (int k0 = 0; k0 < m; k0 += kGK) {
#pragma unroll
    for (int q = 0; q < kGK * T / 256; ++q) {
      const int e = threadIdx.x + 256 * q;
      {
        const int r = e / kGK, k = e % kGK;
        const int row = r0 + r;
        const int kk = k0 + k;
        float v = 0.0f;
        if (row < rows && kk < m) {
          v = X[row * m + kk];
          if (MODE == 0) v -= (float)mean[kk];
        }
        sA[k][r] = v;
      }
      {
        const int k = e / T, c = e % T;
        const int kk = k0 + k, col = c0 + c;
        sB[k][c] = (kk < m && col < m) ? W[(int64_t)kk * m + col] : 0.0f;
      }
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < kGK; ++kk) {
      float a[8], b[8];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float4 av = *reinterpret_cast<const float4*>(&sA[kk][ty * 4 + 64 * h]);
        const float4 bv = *reinterpret_cast<const float4*>(&sB[kk][tx * 4 + 64 * h]);
        a[4 * h] = av.x; a[4 * h + 1] = av.y; a[4 * h + 2] = av.z; a[4 * h + 3] = av.w;
        b[4 * h] = bv.x; b[4 * h + 1] = bv.y; b[4 * h + 2] = bv.z; b[4 * h + 3] = bv.w;
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = r0 + ty * 4 + (i & 3) + 64 * (i >> 2);
    if (row >= rows) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = c0 + tx * 4 + (j & 3) + 64 * (j >> 2);
      if (col < m) O[row * m + col] = (MODE == 0) ? acc[i][j] : B[row * m + col] - acc[i][j];
    }
  }
}

// dst[k] = src[k], k < count (gated: a memcpy node would run in an inactive step too)
__global__ void __launch_bounds__(256)
copy_kernel(const float* __restrict__ src, float* __restrict__ dst, int64_t count, const int* active) {
  if (inactive(active)) return;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride) dst[k] = src[k];
}

int launch_gram(const float* Z, const float* X, int64_t n, int m, const float* shift, const ProjWs& w,
                const int* active, cudaStream_t st) {
  const int T = wide_gram_tile(m);
  const int tiles = (m + T - 1) / T;
  int rb = wide_row_blocks(m);
  const int64_t max_rb = (n + 255) / 256;  // at least 256 rows per block
  if (rb > max_rb) rb = (int)max_rb;
  if (rb < 1) rb = 1;
  int64_t rows_per_block = (n + rb - 1) / rb;
  rows_per_block = (rows_per_block + kGK - 1) / kGK * kGK;
  rb = (int)((n + rows_per_block - 1) / rows_per_block);
  dim3 grid(tiles * tiles, rb);
  if (T == 64) gram_wide_kernel<4><<<grid, 256, 0, st>>>(Z, X, n, m, tiles, rows_per_block, w.fpart, shift, w.shift, active);
  else gram_wide_kernel<8><<<grid, 256, 0, st>>>(Z, X, n, m, tiles, rows_per_block, w.fpart, shift, w.shift, active);
  MDE_LAUNCH_CHECK();
  const int64_t mm = (int64_t)m * m;
  gram_reduce_kernel<<<(unsigned)((mm + 255) / 256), 256, 0, st>>>(w.fpart, rb, mm, w.gram, active);
  MDE_LAUNCH_CHECK();
  return 0;
}

// one fixed-chain product launch: ZY (RES, one product) or Y T and T Z (two)
template <bool RES>
int launch_ns_mm(MmArgs p0, MmArgs p1, int m, double alpha, double beta, double* res_acc, const double* res_prev,
                 double* res_zero, double tol2, int* nsflag, int cur, const int* active, cudaStream_t st) {
  const unsigned z = RES ? 1 : 2;
  if (m <= kWideTileM) {
    const int g = (m + 31) / 32;
    ns_mm_kernel<RES><<<dim3(g, g, z), 256, 0, st>>>(p0, p1, m, alpha, beta, res_acc, res_prev, res_zero, tol2,
                                                      nsflag, cur, active);
  } else {
    const int g = (m + kDT - 1) / kDT;
    ns_dmma_kernel<RES><<<dim3(g, g, z), 128, 0, st>>>(p0, p1, m, alpha, beta, res_acc, res_prev, res_zero, tol2,
                                                        nsflag, cur, active);
  }
  MDE_LAUNCH_CHECK();
  return 0;
}

template <int MODE>
int launch_rowmat_wide(const float* X, float* Y, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st) {
  const int mp = (m + 31) / 32 * 32;
  const size_t smem = sizeof(float) * (32 * (mp + 1) + 16 * mp);  // <= 48.1 KB at mp = 256
  static bool attr[2] = {false, false};
  if (!attr[MODE]) {
    MDE_CUDA_TRY(cudaFuncSetAttribute(rowmat_wide_kernel<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    attr[MODE] = true;
  }
  int64_t tiles = (n + 31) / 32;
  int nb = (int)(tiles < (int64_t)kNumSMs * 4 ? tiles : (int64_t)kNumSMs * 4);
  if (nb < 1) nb = 1;
  rowmat_wide_kernel<MODE><<<nb, 256, smem, st>>>(X, Y, n, m, mp, w.mean, w.wf, active);
  MDE_LAUNCH_CHECK();
  return 0;
}

// m > 256, in chunks of the rows the fpart region holds (16 m of them, or more; the Gram has been reduced by now):
// MODE 0 Y = (X - mu) W through fpart and a copy back (Y may be X), MODE 1 Y -= X W (through fpart when Y is X)
template <int MODE>
int launch_rowgemm(const float* X, float* Y, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st) {
  const int64_t chunk = wide_fpart_floats(m) / m / 128 * 128;
  const bool staged = (const float*)Y == X;
  for (int64_t r0 = 0; r0 < n; r0 += chunk) {
    const int64_t rows = (n - r0 < chunk) ? n - r0 : chunk;
    const float* Xc = X + r0 * m;
    float* Yc = Y + r0 * m;
    float* O = staged ? w.fpart : Yc;
    dim3 grid((unsigned)((m + 127) / 128), (unsigned)((rows + 127) / 128));
    rowgemm_kernel<MODE><<<grid, 256, 0, st>>>(Xc, Yc, O, (int)rows, m, w.mean, w.wf, active);
    MDE_LAUNCH_CHECK();
    if (staged) {
      const int64_t count = rows * m;
      int nb = (int)((count + 1023) / 1024);
      if (nb > kNumSMs * 8) nb = kNumSMs * 8;
      copy_kernel<<<nb, 256, 0, st>>>(w.fpart, Yc, count, active);
      MDE_LAUNCH_CHECK();
    }
  }
  return 0;
}

}  // namespace

namespace mde {

int enqueue_project_standardized_wide(float* X, int64_t n, int m, const ProjWs& w, const int* active, cudaStream_t st) {
  if (!proj_wide(m) || !w.fpart) return MDE_E_UNSUPPORTED;
  int rc;
  // above m = 256 the mean is summed around s as well: an fp32 sum of raw columns 1000 standard deviations off-centre
  // misses mu by ~1e-5 sigma, and A = G_s / n - (mu - s)(mu - s)^T takes that error times |mu - s|
  if ((rc = enqueue_colmean_wide(X, n, m, w, active, st, m > kWideTileM ? X : nullptr))) return rc;
  if ((rc = launch_gram(X, X, n, m, X, w, active, st))) return rc;
  const int64_t mm = (int64_t)m * m;
  double* Yb[2] = {w.ns, w.ns + mm};
  double* Zb[2] = {w.ns + 2 * mm, w.ns + 3 * mm};
  double* T = w.ns + 4 * mm;
  ns_init_kernel<<<1, 1024, 0, st>>>(w.gram, w.mean, w.shift, n, m, Yb[0], Zb[0], w.scal, w.nsflag, w.status, active);
  MDE_LAUNCH_CHECK();
  const double tol = 1e-9 * (double)m, tol2 = tol * tol;
  for (int it = 0; it < kWideNsIters; ++it) {
    const int cur = it & 1, nxt = cur ^ 1;
    double* res = w.scal + 1 + it % 3;
    const double* res_prev = it ? w.scal + 1 + (it - 1) % 3 : nullptr;
    double* res_next = w.scal + 1 + (it + 1) % 3;
    MmArgs zy = {Zb[cur], Yb[cur], T}, none = {nullptr, nullptr, nullptr};
    if ((rc = launch_ns_mm<true>(zy, none, m, -0.5, 1.5, res, res_prev, nullptr, tol2, w.nsflag, cur, active, st))) return rc;
    MmArgs yt = {Yb[cur], T, Yb[nxt]}, tz = {T, Zb[cur], Zb[nxt]};
    if ((rc = launch_ns_mm<false>(yt, tz, m, 1.0, 0.0, nullptr, res_prev, res_next, tol2, w.nsflag, cur, active, st))) return rc;
  }
  ns_finish_kernel<<<(unsigned)((mm + 255) / 256), 256, 0, st>>>(w.ns, mm, w.scal, w.nsflag, kWideNsIters & 1,
                                                                w.scal + 1 + (kWideNsIters - 1) % 3, tol2, w.wf, w.status, active);
  MDE_LAUNCH_CHECK();
  return m <= kWideTileM ? launch_rowmat_wide<0>(X, X, n, m, w, active, st) : launch_rowgemm<0>(X, X, n, m, w, active, st);
}

int enqueue_tangent_standardized_wide(const float* X, float* Z, int64_t n, int m, const ProjWs& w,
                                      const int* active, cudaStream_t st) {
  if (!proj_wide(m) || !w.fpart) return MDE_E_UNSUPPORTED;
  int rc;
  if ((rc = launch_gram(Z, X, n, m, nullptr, w, active, st))) return rc;
  const int64_t mm = (int64_t)m * m;
  tangent_mat_kernel<<<(unsigned)((mm + 255) / 256), 256, 0, st>>>(w.gram, mm, 1.0 / (double)n, w.wf, active);
  MDE_LAUNCH_CHECK();
  return m <= kWideTileM ? launch_rowmat_wide<1>(X, Z, n, m, w, active, st) : launch_rowgemm<1>(X, Z, n, m, w, active, st);
}

}  // namespace mde
