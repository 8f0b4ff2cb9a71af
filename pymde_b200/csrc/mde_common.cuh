// mde_common.cuh -- shared device helpers for the H100 (sm_90a) MDE hot path.
//
// Distortion functions follow cvxgrp/pymde v0.2.1 pymde/functions/penalties.py:112-400 and
// pymde/functions/losses.py:61-239; the reference differentiates them with torch autograd,
// here f and f' are evaluated in closed form (same conventions at the kinks: sign(0) = 0,
// max() tie -> averaged slope).  All arithmetic is fp32 like the reference; reductions
// that the reference does in fp32 (mean, dot) are accumulated in fp64 here.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/mde_b200.h"

namespace mde {

extern unsigned long long g_launch_count;  // host-side counter (mde_launch_count)

#define MDE_CUDA_TRY(expr)                         \
  do {                                             \
    cudaError_t _e = (expr);                       \
    if (_e != cudaSuccess) return (int)_e;         \
  } while (0)

#define MDE_LAUNCH_CHECK()                         \
  do {                                             \
    ++::mde::g_launch_count;                       \
    cudaError_t _e = cudaPeekAtLastError();        \
    if (_e != cudaSuccess) return (int)_e;         \
  } while (0)

constexpr int kNumSMs = 132;  // H100 SXM; the persistent grids assume it (a 114-SM PCIe part runs a partial second wave)
constexpr unsigned kFull = 0xffffffffu;

struct FnDev {
  int fn_att, fn_rep;
  float a0, a1, a2;
  float r0, r1, r2;
  int push_pull;
};

inline FnDev to_dev(const mde_fn_t& f) {
  FnDev d;
  d.fn_att = f.fn_att; d.fn_rep = f.fn_rep;
  d.a0 = f.att[0]; d.a1 = f.att[1]; d.a2 = f.att[2];
  d.r0 = f.rep[0]; d.r1 = f.rep[1]; d.r2 = f.rep[2];
  d.push_pull = f.push_pull;
  return d;
}

__device__ __forceinline__ float signf(float x) { return (float)(x > 0.0f) - (float)(x < 0.0f); }

// d^e and d^(e-1); the common exponents avoid powf.
__device__ __forceinline__ void pow_pair(float d, float e, float& de, float& dem1) {
  if (e == 1.0f) { de = d; dem1 = 1.0f; }
  else if (e == 2.0f) { de = d * d; dem1 = d; }
  else if (e == 1.5f) { float s = sqrtf(d); de = d * s; dem1 = s; }
  else if (e == 3.0f) { de = d * d * d; dem1 = d * d; }
  else if (e == 0.5f) { float s = sqrtf(d); de = s; dem1 = 1.0f / s; }
  else { de = powf(d, e); dem1 = powf(d, e - 1.0f); }
}

// f(d) and f'(d) for one function id known at COMPILE time.  a = weight | deviation,
// b = second per-edge array (WeightedQuadratic weights).
template <int FN>
__device__ __forceinline__ void eval_fn_t(float s0, float s1, float d, float a, float b, float& f, float& fp) {
  if constexpr (FN == MDE_FN_P_LINEAR) {
    f = a * d; fp = a;
  }
  else if constexpr (FN == MDE_FN_P_QUADRATIC) {
    f = a * d * d; fp = 2.0f * a * d;
  }
  else if constexpr (FN == MDE_FN_P_CUBIC) {
    f = a * d * d * d; fp = 3.0f * a * d * d;
  }
  else if constexpr (FN == MDE_FN_P_POWER) {
    float de, dem1; pow_pair(d, s0, de, dem1);
      f = a * de; fp = a * s0 * dem1;
  }
  else if constexpr (FN == MDE_FN_P_HUBER) {
    if (d < s0) { f = a * 0.5f * d * d; fp = a * d; }
      else { f = a * s0 * (d - 0.5f * s0); fp = a * s0; }
  }
  else if constexpr (FN == MDE_FN_P_LOGISTIC) {
    float z = s1 * (d - s0);
      f = a * (fmaxf(z, 0.0f) + log1pf(expf(-fabsf(z))));
      fp = a * s1 / (1.0f + expf(-z));
  }
  else if constexpr (FN == MDE_FN_P_LOG1P) {
    float de, dem1; pow_pair(d, s0, de, dem1);
      f = a * log1pf(de); fp = a * s0 * dem1 / (1.0f + de);
  }
  else if constexpr (FN == MDE_FN_P_LOG) {
    float de, dem1; pow_pair(d, s0, de, dem1);
      f = a * logf(-expm1f(-de)); fp = a * s0 * dem1 / expm1f(de);
  }
  else if constexpr (FN == MDE_FN_P_INVPOWER) {
    float de, dem1; pow_pair(d, s0, de, dem1);
      float aw = fabsf(a);
      f = aw / de; fp = -aw * s0 / (de * d);
  }
  else if constexpr (FN == MDE_FN_P_LOGRATIO) {
    float de, dem1; pow_pair(d, s0, de, dem1);
      f = a * logf(de / (1.0f + de)); fp = a * s0 / (d * (1.0f + de));
  }
  else if constexpr (FN == MDE_FN_L_ABSOLUTE) {
    f = fabsf(a - d); fp = signf(d - a);
  }
  else if constexpr (FN == MDE_FN_L_QUADRATIC) {
    float r = a - d; f = r * r; fp = 2.0f * (d - a);
  }
  else if constexpr (FN == MDE_FN_L_WEIGHTED_QUADRATIC) {
    float r = a - d; f = b * r * r; fp = 2.0f * b * (d - a);
  }
  else if constexpr (FN == MDE_FN_L_HUBER) {
    // branch-free, same values: c = clamp(d - a, -s0, s0); |e| < s0: f = e (2e - e) = e^2, f' = 2e;
    // otherwise f = s0 (2|e| - s0), f' = 2 s0 sign(e)   (losses.py:101-125)
    const float e = d - a;
    const float c = fminf(fmaxf(e, -s0), s0);
    f = c * (2.0f * e - c);
    fp = 2.0f * c;
  }
  else if constexpr (FN == MDE_FN_L_CUBIC) {
    float r = fabsf(a - d); f = r * r * r; fp = 3.0f * r * r * signf(d - a);
  }
  else if constexpr (FN == MDE_FN_L_POWER) {
    float r = fabsf(a - d); float re, rem1; pow_pair(r, s0, re, rem1);
      f = re; fp = s0 * rem1 * signf(d - a);
  }
  else if constexpr (FN == MDE_FN_L_LOGISTIC) {
    // naive log(1 + exp(r)) as written in losses.py:184-186
      float r = fabsf(a - d); float er = expf(r);
      f = logf(1.0f + er); fp = er / (1.0f + er) * signf(d - a);
  }
  else if constexpr (FN == MDE_FN_L_FRACTIONAL) {
    float u = a / d, v = d / a;
      f = fmaxf(u, v) - 1.0f;
      float du = -a / (d * d), dv = 1.0f / a;
      fp = (v > u) ? dv : ((u > v) ? du : 0.5f * (du + dv));
  }
  else if constexpr (FN == MDE_FN_L_SOFT_FRACTIONAL) {
    float u = s0 * a / d, v = s0 * d / a;
      float mx = fmaxf(u, v);
      float lse = isinf(mx) ? mx : mx + logf(expf(u - mx) + expf(v - mx));
      float inv_gamma = 1.0f / s0;
      f = inv_gamma * (lse - (0.69314718f + s0));
      float pu = expf(u - lse), pv = expf(v - lse);
      fp = (inv_gamma * s0) * (pu * (-a / (d * d)) + pv * (1.0f / a));
  }
  else { f = 0.0f; fp = 0.0f; }
}

// Run-time function id: ONE out-of-line copy of the whole table (keeps the generic kernels small).
static __device__ __noinline__ float2 eval_fn_rt(int fn, float s0, float s1, float d, float a, float b) {
  float f, fp;  // returned by value: references into a non-inlined call would live in local memory
  switch (fn) {
#define MDE_CASE(X) case X: eval_fn_t<X>(s0, s1, d, a, b, f, fp); break;
    MDE_CASE(MDE_FN_P_LINEAR) MDE_CASE(MDE_FN_P_QUADRATIC) MDE_CASE(MDE_FN_P_CUBIC) MDE_CASE(MDE_FN_P_POWER)
    MDE_CASE(MDE_FN_P_HUBER) MDE_CASE(MDE_FN_P_LOGISTIC) MDE_CASE(MDE_FN_P_LOG1P) MDE_CASE(MDE_FN_P_LOG)
    MDE_CASE(MDE_FN_P_INVPOWER) MDE_CASE(MDE_FN_P_LOGRATIO) MDE_CASE(MDE_FN_L_ABSOLUTE) MDE_CASE(MDE_FN_L_QUADRATIC)
    MDE_CASE(MDE_FN_L_WEIGHTED_QUADRATIC) MDE_CASE(MDE_FN_L_HUBER) MDE_CASE(MDE_FN_L_CUBIC) MDE_CASE(MDE_FN_L_POWER)
    MDE_CASE(MDE_FN_L_LOGISTIC) MDE_CASE(MDE_FN_L_FRACTIONAL) MDE_CASE(MDE_FN_L_SOFT_FRACTIONAL)
#undef MDE_CASE
    default: f = 0.0f; fp = 0.0f; break;
  }
  return make_float2(f, fp);
}

// f_k(d) and f'_k(d) of edge k.  FA/FR >= 0: function ids fixed at compile time (hot combinations);
// FA < 0: run-time table.  PushAndPull picks attractive/repulsive by weight sign (penalties.py:390).
template <int FA, int FR>
__device__ __forceinline__ void edge_f_fp(const FnDev& fn, float d, float a, float b, float& f, float& fp) {
  if constexpr (FA < 0) {
    const bool rep = fn.push_pull && !(a >= 0.0f);
    const float2 r = rep ? eval_fn_rt(fn.fn_rep, fn.r0, fn.r1, d, a, b) : eval_fn_rt(fn.fn_att, fn.a0, fn.a1, d, a, b);
    f = r.x; fp = r.y;
  } else if constexpr (FA == FR) {
    eval_fn_t<FA>(fn.a0, fn.a1, d, a, b, f, fp);
  } else {
    if (!(a >= 0.0f)) eval_fn_t<FR>(fn.r0, fn.r1, d, a, b, f, fp);
    else eval_fn_t<FA>(fn.a0, fn.a1, d, a, b, f, fp);
  }
}

// Per-edge distortion f_k(d) and gradient coefficient g_k = f'_k(d) / (p d), with the
// reference's guard: non-finite g -> 1.0 (pymde/average_distortion.py:55-62; it only fires
// when d = 0, where the difference vector is 0 too).
template <int FA, int FR>
__device__ __forceinline__ void edge_coeff(const FnDev& fn, float d, float a, float b, float inv_p,
                                           float& f, float& g) {
  float fp;
  edge_f_fp<FA, FR>(fn, d, a, b, f, fp);
  float gp = fp * inv_p;
  g = gp / d;
  if (!isfinite(g)) g = 1.0f;
}

template <int FA, int FR>
__device__ __forceinline__ void edge_value(const FnDev& fn, float d, float a, float b, float& f) {
  float fp;
  edge_f_fp<FA, FR>(fn, d, a, b, f, fp);
}

// ------------------------------------------------------------------------------------------
// fast path for the recipe default PushAndPull(Log1p(1.5), Log(1.0)) (pymde/recipes.py:224-225):
// MUFU approximations (rsqrt / sqrt / rcp / lg2 / ex2, <= 2 ulp each) instead of the IEEE
// sequences.  The kernel is instruction-issue bound, and only the
// SUM of the per-edge losses has to agree with the reference to 1e-5: a 1e-7 absolute error per edge
// is far inside that.  Inputs: squared distance d2.  Outputs: f_k and g_k = f'_k / (p d).
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float fast_rsqrt(float x) { float y; asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_sqrt(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_rcp(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_lg2(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float fast_ex2(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }

__device__ __forceinline__ void edge_coeff_fast_log1p_log(float d2, float w, float inv_p, float& f, float& g) {
  const float kLn2 = 0.69314718056f, kLog2e = 1.44269504089f;
  const float rs = fast_rsqrt(d2);          // 1/d  (inf at d2 = 0; masked by the caller)
  const float d = (d2 > 0.0f) ? d2 * rs : 0.0f;  // 0 * inf would be NaN
  if (w >= 0.0f) {                          // attractive: w log1p(d^1.5)
    const float sd = fast_sqrt(d);
    const float de = d * sd;
    const float one_p = 1.0f + de;
    f = w * kLn2 * fast_lg2(one_p);
    g = w * (1.5f * inv_p) * sd * rs * fast_rcp(one_p);
  } else {                                  // repulsive: w log(1 - exp(-d)),  f' = w / expm1(d)
    const float em = fast_ex2(-d * kLog2e);                                      // e^-d
    float one_m = 1.0f - em;                                                     // 1 - e^-d
    const float series = d * (1.0f - d * (0.5f - d * (0.16666667f - d * 0.041666668f)));
    one_m = (d < 0.0625f) ? series : one_m;                                      // no cancellation for small d
    f = w * kLn2 * fast_lg2(one_m);
    g = w * inv_p * rs * em * fast_rcp(one_m);
  }
}

// ------------------------------------------------------------------------------------------
// reductions
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(kFull, v, off);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, off));
  return v;
}

// Block-wide sum of K doubles per thread (blockDim.x multiple of 32, <= 1024).  Result valid
// in thread 0.  `smem` needs K * 32 doubles.  Deterministic for a fixed launch shape.
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double* smem) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = warp_sum(v[k]);
  __syncthreads();
  if (lane == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) smem[k * 32 + w] = v[k];
  }
  __syncthreads();
  if (w == 0) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
      double x = (lane < nw) ? smem[k * 32 + lane] : 0.0;
      v[k] = warp_sum(x);
    }
  }
}

// vector reductions without return value (SASS: REDG.E.ADD.F32x2 / F32x4), sm_90+.
__device__ __forceinline__ void red_add(float* a, float x) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(a), "f"(x) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* a, float x, float y) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(a), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ void red_add_v4(float* a, float x, float y, float z, float w) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(a), "f"(x), "f"(y), "f"(z), "f"(w)
               : "memory");
}

inline int ceil_div_i64(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

}  // namespace mde
