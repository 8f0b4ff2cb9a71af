// mde_logic.h -- scalar control logic of the projected L-BFGS solve, as resumable state
// machines that run in ONE thread on the device (and, for unit tests, on the host).
//
// Reference (cvxgrp/pymde v0.2.1):
//   _strong_wolfe / _cubic_interpolate   pymde/lbfgs.py:16-253
//   LBFGS.step direction update          pymde/lbfgs.py:461-531
// The reference runs these as Python control flow with one host<->device sync per scalar
// (SURVEY section 2.1).  Here every scalar lives in device memory: the line search is a state
// machine advanced once per trial evaluation, and the two-loop recursion is carried out on
// the Gram matrix of the history ("vector-free" form) so that it needs no n*m-sized passes.
//
// Scalar types follow the reference: f and t are doubles (Python floats) except that an
// interpolated t is an fp32 value (0-dim fp32 tensor); directional derivatives are fp32.
#pragma once
#include <math.h>
#include <stdint.h>

#ifdef __CUDACC__
#define MDE_HD __host__ __device__
#else
#define MDE_HD
#endif

namespace mde {

constexpr int kMaxMemory = 32;          // L-BFGS history pairs supported on device
constexpr int kSlots = kMaxMemory + 1;  // one spare slot for the candidate pair

// ---------------------------------------------------------------------------------------
// strong-Wolfe line search
// ---------------------------------------------------------------------------------------
enum LsPhase { LS_BACKOFF = 0, LS_BRACKET = 1, LS_ZOOM = 2, LS_FALLBACK = 3, LS_FINAL0 = 4, LS_DONE = 5 };

struct LsState {
  int phase;
  int ls_iter;
  int backoff;        // evaluations spent in the initial NaN/Inf back-off
  int func_evals;
  int done;           // Wolfe conditions met (reference variable `done`)
  int insuf_progress;
  int nbracket;       // 1 or 2
  int low_pos, high_pos;
  int error;          // 0 ok, MDE_E_NAN-like code otherwise
  double t;           // step to evaluate next / last evaluated
  double t_prev, f_prev;
  float gtd_prev;
  double bt[2], bf[2];
  float bg[2];
  double f0;          // loss at t = 0
  float gtd0;         // g.d at t = 0
  float d_norm;       // max |d|
  double f_new;       // last evaluated loss
  float gtd_new;
  double t_accept, f_accept;
};

MDE_HD inline bool ls_isnan(double x) { return x != x; }
MDE_HD inline bool ls_isinf(double x) { return !ls_isnan(x) && ls_isnan(x - x); }

// lbfgs.py:16-41.  x1,x2,f1,f2 doubles; g1,g2 fp32.
MDE_HD inline double ls_cubic(double x1, double f1, float g1, double x2, double f2, float g2,
                              bool has_bounds, double lo_b, double hi_b) {
  double xmin_bound, xmax_bound;
  if (has_bounds) { xmin_bound = lo_b; xmax_bound = hi_b; }
  else if (x1 <= x2) { xmin_bound = x1; xmax_bound = x2; }
  else { xmin_bound = x2; xmax_bound = x1; }
  float d1 = g1 + g2 - (float)(3.0 * (f1 - f2) / (x1 - x2));
  float d2_square = d1 * d1 - g1 * g2;
  if (d2_square >= 0.0f) {
    float d2 = sqrtf(d2_square);
    float min_pos;
    if (x1 <= x2) min_pos = (float)x2 - (float)(x2 - x1) * ((g2 + d2 - d1) / (g2 - g1 + 2.0f * d2));
    else min_pos = (float)x1 - (float)(x1 - x2) * ((g1 + d2 - d1) / (g1 - g2 + 2.0f * d2));
    // python: min(max(min_pos, xmin_bound), xmax_bound)
    double lo = (xmin_bound > (double)min_pos) ? xmin_bound : (double)min_pos;
    return (xmax_bound < lo) ? xmax_bound : lo;
  }
  return (xmin_bound + xmax_bound) / 2.0;
}

// Armijo right-hand side as the reference forms it: fp32(f + fp32(fp32(c1*t) * gtd))
MDE_HD inline float ls_armijo_rhs(double f, double t, float gtd) {
  return (float)f + ((float)(1e-4 * t)) * gtd;
}

MDE_HD inline void ls_begin(LsState& L, double t0, double f0, float gtd0, float d_norm) {
  L.phase = LS_BACKOFF; L.ls_iter = 0; L.backoff = 0; L.func_evals = 0; L.done = 0;
  L.insuf_progress = 0; L.nbracket = 0; L.low_pos = 0; L.high_pos = 1; L.error = 0;
  L.t = t0; L.t_prev = 0.0; L.f_prev = f0; L.gtd_prev = gtd0;
  L.f0 = f0; L.gtd0 = gtd0; L.d_norm = d_norm;
  L.f_new = f0; L.gtd_new = gtd0; L.t_accept = 0.0; L.f_accept = f0;
}

namespace detail {

MDE_HD inline void ls_complete(LsState& L) {
  L.t_accept = L.t; L.f_accept = L.f_new; L.phase = LS_DONE;
}

// lbfgs.py:239-249
MDE_HD inline void ls_fallback_next(LsState& L);
MDE_HD inline void ls_fallback_end(LsState& L) {
  if (ls_isnan(L.f_new)) { L.t = 0.0; L.phase = LS_FINAL0; return; }  // evaluate at t = 0
  ls_complete(L);
}
MDE_HD inline void ls_fallback_next(LsState& L) {
  if (L.t > 1e-8) { L.t = L.t * 0.8; L.phase = LS_FALLBACK; return; }  // evaluate
  ls_fallback_end(L);
}

// lbfgs.py:227-251
MDE_HD inline void ls_finish(LsState& L) {
  bool failed = ls_isnan(L.f_new);
  if (L.low_pos < L.nbracket) { L.t = L.bt[L.low_pos]; L.f_new = L.bf[L.low_pos]; }
  else { L.t = 1.0; failed = true; }
  if (failed) { ls_fallback_next(L); return; }
  ls_fallback_end(L);
}

// head of the zoom loop, lbfgs.py:147-181: either finish or set the next trial step
MDE_HD inline void ls_zoom_next(LsState& L) {
  if (L.done || L.ls_iter >= 25) { ls_finish(L); return; }
  double b0 = L.bt[0], b1 = L.bt[1];
  if (fabs(b1 - b0) * (double)L.d_norm < 1e-9) { ls_finish(L); return; }
  double t = ls_cubic(b0, L.bf[0], L.bg[0], b1, L.bf[1], L.bg[1], false, 0.0, 0.0);
  double bmax = b0 > b1 ? b0 : b1, bmin = b0 < b1 ? b0 : b1;
  double eps = 0.1 * (bmax - bmin);
  double m1 = bmax - t, m2 = t - bmin;
  if ((m1 < m2 ? m1 : m2) < eps) {
    if (L.insuf_progress || t >= bmax || t <= bmin) {
      if (fabs(t - bmax) < fabs(t - bmin)) t = bmax - eps; else t = bmin + eps;
      L.insuf_progress = 0;
    } else {
      L.insuf_progress = 1;
    }
  } else {
    L.insuf_progress = 0;
  }
  L.t = t; L.ls_iter += 1; L.phase = LS_ZOOM;  // evaluate
}

MDE_HD inline void ls_zoom_begin(LsState& L) {
  L.insuf_progress = 0;
  double last = L.bf[L.nbracket - 1];
  if (L.bf[0] <= last) { L.low_pos = 0; L.high_pos = 1; } else { L.low_pos = 1; L.high_pos = 0; }
  ls_zoom_next(L);
}

// bracketing loop body with a fresh (f_new, gtd_new) at L.t, lbfgs.py:87-139
MDE_HD inline void ls_bracket_check(LsState& L) {
  const double t = L.t, f_new = L.f_new;
  const float gtd_new = L.gtd_new;
  if (L.ls_iter < 25) {
    if (f_new > (double)ls_armijo_rhs(L.f0, t, L.gtd0) || (L.ls_iter > 1 && f_new >= L.f_prev)) {
      L.nbracket = 2; L.bt[0] = L.t_prev; L.bt[1] = t; L.bf[0] = L.f_prev; L.bf[1] = f_new;
      L.bg[0] = L.gtd_prev; L.bg[1] = gtd_new;
      ls_zoom_begin(L); return;
    }
    if (fabsf(gtd_new) <= -0.9f * L.gtd0) {
      L.nbracket = 1; L.bt[0] = t; L.bf[0] = f_new; L.bg[0] = gtd_new; L.bt[1] = t; L.bf[1] = f_new; L.bg[1] = gtd_new;
      L.done = 1;
      ls_zoom_begin(L); return;
    }
    if (gtd_new >= 0.0f) {
      L.nbracket = 2; L.bt[0] = L.t_prev; L.bt[1] = t; L.bf[0] = L.f_prev; L.bf[1] = f_new;
      L.bg[0] = L.gtd_prev; L.bg[1] = gtd_new;
      ls_zoom_begin(L); return;
    }
    double min_step = t + 0.01 * (t - L.t_prev);
    double max_step = t * 10.0;
    double tn = ls_cubic(L.t_prev, L.f_prev, L.gtd_prev, t, f_new, gtd_new, true, min_step, max_step);
    L.t_prev = t; L.f_prev = f_new; L.gtd_prev = gtd_new;
    L.t = tn; L.ls_iter += 1; L.phase = LS_BRACKET;  // evaluate
    return;
  }
  // ls_iter == max_ls, lbfgs.py:136-139
  L.nbracket = 2; L.bt[0] = 0.0; L.bt[1] = t; L.bf[0] = L.f0; L.bf[1] = f_new; L.bg[0] = L.gtd0; L.bg[1] = gtd_new;
  ls_zoom_begin(L);
}

}  // namespace detail

// Feed the result of evaluating at L.t.  `grad_finite` = no NaN/Inf in the gradient.
// Afterwards either L.phase == LS_DONE (t_accept / f_accept / error set) or L.t holds the
// next step to evaluate.
MDE_HD inline void ls_on_result(LsState& L, double f_new, float gtd_new, bool grad_finite) {
  L.f_new = f_new; L.gtd_new = gtd_new; L.func_evals += 1;
  switch (L.phase) {
    case LS_BACKOFF: {  // lbfgs.py:59-80
      bool bad = ls_isnan(f_new) || ls_isinf(f_new) || !grad_finite;
      L.backoff += 1;
      if (bad) {
        L.t = L.t * 0.5;
        if (L.backoff >= 10) { L.error = 1; L.t = 0.0; L.t_accept = 0.0; L.f_accept = L.f0; L.phase = LS_DONE; }
        return;  // evaluate again at the halved step
      }
      L.func_evals = 1;
      L.t_prev = 0.0; L.f_prev = L.f0; L.gtd_prev = L.gtd0; L.ls_iter = 0;
      L.phase = LS_BRACKET;
      detail::ls_bracket_check(L);
      return;
    }
    case LS_BRACKET: detail::ls_bracket_check(L); return;
    case LS_ZOOM: {  // lbfgs.py:188-224
      const double t = L.t;
      if (ls_isnan(f_new) || f_new > (double)ls_armijo_rhs(L.f0, t, L.gtd0) || f_new >= L.bf[L.low_pos]) {
        L.bt[L.high_pos] = t; L.bf[L.high_pos] = f_new; L.bg[L.high_pos] = gtd_new;
        if (L.bf[0] <= L.bf[1]) { L.low_pos = 0; L.high_pos = 1; } else { L.low_pos = 1; L.high_pos = 0; }
      } else {
        if (fabsf(gtd_new) <= -0.9f * L.gtd0) {
          L.done = 1;
        } else if ((double)gtd_new * (L.bt[L.high_pos] - L.bt[L.low_pos]) >= 0.0) {
          L.bt[L.high_pos] = L.bt[L.low_pos]; L.bf[L.high_pos] = L.bf[L.low_pos]; L.bg[L.high_pos] = L.bg[L.low_pos];
        }
        L.bt[L.low_pos] = t; L.bf[L.low_pos] = f_new; L.bg[L.low_pos] = gtd_new;
      }
      detail::ls_zoom_next(L);
      return;
    }
    case LS_FALLBACK: {  // lbfgs.py:240-246
      if (ls_isnan(f_new)) { detail::ls_fallback_next(L); return; }
      if (f_new < (double)ls_armijo_rhs(L.f0, L.t, L.gtd0)) { detail::ls_fallback_end(L); return; }
      detail::ls_fallback_next(L);
      return;
    }
    case LS_FINAL0: detail::ls_complete(L); return;
    default: return;
  }
}

// ---------------------------------------------------------------------------------------
// L-BFGS history in Gram form
// ---------------------------------------------------------------------------------------
struct LbfgsState {
  // Gram matrices in LOGICAL order: SY[i][j] = s_i . y_j, YY[i][j] = y_i . y_j
  double SY[kMaxMemory][kMaxMemory];
  double YY[kMaxMemory][kMaxMemory];
  double H_diag;
  // coefficients of the new direction d = cg*g + sum_j cs[j]*S[order[j]] + cy[j]*Y[order[j]]
  double cg, cs[kSlots], cy[kSlots];
  int n_iter;            // state["n_iter"] (0 after reset)
  int count;             // pairs held
  int cand;              // free physical slot receiving the candidate pair
  int memory;            // history_size
  int order[kSlots + 1]; // logical (oldest..newest) -> physical slot of S / Y (padded to an even count)
};

MDE_HD inline void lbfgs_reset(LbfgsState& B, int memory) {
  B.n_iter = 0; B.count = 0; B.cand = 0; B.memory = memory; B.H_diag = 1.0;
  for (int i = 0; i < kSlots; ++i) B.order[i] = i;
  B.cg = -1.0;
}

// Dots delivered by the vector pass, indexed by LOGICAL pair j (before the update):
//   ys, yy           : candidate y.s, y.y
//   sc_g, yc_g       : candidate s.g, y.g  (g = current gradient)
//   sj_yc[j], yj_yc[j], sc_yj[j], sj_g[j], yj_g[j]
// SY / YY point at kMaxMemory x kMaxMemory logical-order matrices (shared or global memory).
// Mirrors lbfgs.py:467-507: accept the pair iff ys > 1e-10, evict the oldest when full,
// H_diag = ys / yy, then the two-loop recursion -- carried out on dot products only.
MDE_HD inline void lbfgs_direction(LbfgsState& B, double (*SY)[kMaxMemory], double (*YY)[kMaxMemory],
                                   double ys, double yy, double sc_g, double yc_g,
                                   double* sj_yc, double* yj_yc, double* sc_yj,
                                   double* sj_g, double* yj_g) {
  B.n_iter += 1;
  if (B.n_iter == 1) {  // lbfgs.py:461-466: steepest descent
    B.count = 0; B.H_diag = 1.0; B.cg = -1.0;
    return;
  }
  int h = B.count;
  if ((float)ys > 1e-10f) {  // fp32 dot in the reference
    const int c = B.cand;
    if (h == B.memory) {  // evict the oldest; its slot becomes the next candidate slot
      int freed = B.order[0];
      for (int j = 1; j < h; ++j) {
        B.order[j - 1] = B.order[j];
        sj_yc[j - 1] = sj_yc[j]; yj_yc[j - 1] = yj_yc[j]; sc_yj[j - 1] = sc_yj[j];
        sj_g[j - 1] = sj_g[j]; yj_g[j - 1] = yj_g[j];
      }
      for (int i = 1; i < h; ++i)
        for (int j = 1; j < h; ++j) { SY[i - 1][j - 1] = SY[i][j]; YY[i - 1][j - 1] = YY[i][j]; }
      h -= 1;
      B.order[h] = c; B.cand = freed;
    } else {
      B.order[h] = c;
      bool used[kSlots];
      for (int i = 0; i < kSlots; ++i) used[i] = false;
      for (int j = 0; j <= h; ++j) used[B.order[j]] = true;
      int f = 0;
      while (f < kSlots - 1 && used[f]) ++f;
      B.cand = f;
    }
    for (int j = 0; j < h; ++j) {
      SY[j][h] = sj_yc[j]; SY[h][j] = sc_yj[j];
      YY[j][h] = yj_yc[j]; YY[h][j] = yj_yc[j];
    }
    SY[h][h] = ys; YY[h][h] = yy;
    sj_g[h] = sc_g; yj_g[h] = yc_g;
    h += 1;
    B.count = h;
    B.H_diag = (double)((float)ys / (float)yy);
  }
  // two-loop recursion in coefficient space (lbfgs.py:488-507)
  double al[kMaxMemory], cc[kMaxMemory];
  for (int i = h - 1; i >= 0; --i) {
    double sq = -sj_g[i];
    for (int j = i + 1; j < h; ++j) sq -= al[j] * SY[i][j];
    al[i] = sq / SY[i][i];
  }
  for (int i = 0; i < h; ++i) {
    double yq = -yj_g[i];
    for (int j = 0; j < h; ++j) yq -= al[j] * YY[i][j];
    double yr = B.H_diag * yq;
    for (int j = 0; j < i; ++j) yr += cc[j] * SY[j][i];
    double be = yr / SY[i][i];
    cc[i] = al[i] - be;
  }
  B.cg = -B.H_diag;
  for (int j = 0; j < h; ++j) { B.cs[j] = cc[j]; B.cy[j] = -B.H_diag * al[j]; }
}

// ---------------------------------------------------------------------------------------
// exact k-nearest-neighbour search (mde_knn.cu): candidate slices
// ---------------------------------------------------------------------------------------
// One CTA per (query tile, candidate slice), one CTA per SM.  When the q_tiles query tiles leave SMs idle, the sweep
// over the c_tiles candidate tiles is split into S slices: as many as keep q_tiles S within one wave of num_sms CTAs,
// at most one candidate tile per slice and at most max_slices (the merge re-ranks S times the candidates).  S = 1
// once the query tiles fill the SMs.
MDE_HD inline int knn_slices(int64_t q_tiles, int64_t c_tiles, int num_sms, int max_slices) {
  if (q_tiles < 1 || q_tiles >= num_sms) return 1;
  int64_t s = num_sms / q_tiles;
  if (s > c_tiles) s = c_tiles;
  if (s > max_slices) s = max_slices;
  return s < 1 ? 1 : (int)s;
}

}  // namespace mde
