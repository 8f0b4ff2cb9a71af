/*
 * mde_b200.h -- C ABI of the H100-native (sm_90a) MDE hot path (libmde_b200.so).
 *
 * The reference (cvxgrp/pymde v0.2.1) has no FFI of its own: its hot path is a chain of
 * torch ops behind Python call boundaries.  Each entry point below replaces one of those
 * boundaries; the "replaces" note cites the reference file:line.  A maintainer binds them
 * with ctypes (INTEGRATION.md shows the stub); pymde_b200/_lib.py is that binding.
 *
 * Conventions
 *  - every function returns 0 on success, a positive cudaError_t on a CUDA failure, or a
 *    negative MDE_E_* code; no C++ exception or exit() crosses this boundary;
 *  - all array pointers are DEVICE pointers owned by the caller (torch-allocated) unless
 *    the name ends in _host; the library never frees caller memory and never mutates the
 *    caller's int64 edge list;
 *  - `stream` is a cudaStream_t passed as void*; all work is enqueued on it and no call
 *    synchronises the device unless documented ("blocking");
 *  - matrices are row-major contiguous float32: X[n_items][m].
 */
#ifndef MDE_B200_H
#define MDE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MDE_ABI_VERSION 1

/* error codes (negative; positive values are cudaError_t) */
#define MDE_E_INVALID   (-1)  /* bad argument */
#define MDE_E_UNSUPPORTED (-2) /* combination not built (e.g. Standardized with m > 32) */
#define MDE_E_NAN       (-3)  /* line search: function/gradient stayed NaN/Inf (lbfgs.py:70-80) */
#define MDE_E_ALLOC     (-4)
#define MDE_E_COMM      (-5)  /* multi-GPU: a peer never arrived at the all-reduce handshake (bounded spin) */

/* distortion function ids -- pymde/functions/penalties.py, pymde/functions/losses.py */
enum {
  MDE_FN_P_LINEAR = 1,      /* penalties.py:112 */
  MDE_FN_P_QUADRATIC = 2,   /* :123 */
  MDE_FN_P_CUBIC = 3,       /* :163 */
  MDE_FN_P_POWER = 4,       /* :191  s[0]=exponent */
  MDE_FN_P_HUBER = 5,       /* :205  s[0]=threshold */
  MDE_FN_P_LOGISTIC = 6,    /* :246  s[0]=threshold s[1]=alpha */
  MDE_FN_P_LOG1P = 7,       /* :310  s[0]=exponent */
  MDE_FN_P_LOG = 8,         /* :324  s[0]=exponent */
  MDE_FN_P_INVPOWER = 9,    /* :340  s[0]=exponent */
  MDE_FN_P_LOGRATIO = 10,   /* :356  s[0]=exponent */
  MDE_FN_L_ABSOLUTE = 20,   /* losses.py:166 */
  MDE_FN_L_QUADRATIC = 21,  /* :61 */
  MDE_FN_L_WEIGHTED_QUADRATIC = 22, /* :72  par1 = weights */
  MDE_FN_L_HUBER = 23,      /* :101  s[0]=threshold */
  MDE_FN_L_CUBIC = 24,      /* :128 */
  MDE_FN_L_POWER = 25,      /* :139  s[0]=exponent */
  MDE_FN_L_LOGISTIC = 26,   /* :177 */
  MDE_FN_L_FRACTIONAL = 27, /* :189 */
  MDE_FN_L_SOFT_FRACTIONAL = 28, /* :203  s[0]=gamma */
  MDE_FN_EXTERNAL = 100     /* per-edge g supplied by the caller (arbitrary Python callables) */
};

/* A vector distortion function in table form.  For penalties.PushAndPull (penalties.py:372)
 * push_pull = 1 and edge k uses (fn_att, att) when par0[k] >= 0, else (fn_rep, rep). */
typedef struct mde_fn {
  int32_t fn_att;
  int32_t fn_rep;
  float att[3];
  float rep[3];
  int32_t push_pull;
} mde_fn_t;

/* constraint ids -- pymde/constraints.py */
enum { MDE_CONSTRAINT_CENTERED = 0, MDE_CONSTRAINT_STANDARDIZED = 1, MDE_CONSTRAINT_ANCHORED = 2,
       MDE_CONSTRAINT_CUSTOM = 3 /* caller-defined projections: mde_solver_create_custom only */ };

typedef struct mde_edges mde_edges_t;   /* device-resident edge layout (one shard) */
typedef struct mde_solver mde_solver_t; /* device-resident projected L-BFGS state */

int mde_abi_version(void);
const char* mde_error_string(int code);
/* number of kernels this library has launched since load (bench.py `gpu_launches`). */
uint64_t mde_launch_count(void);

/* ---------------------------------------------------------------------------------------
 * Edge layout.  Replaces MDE.__init__'s `_lhs/_rhs` index views (pymde/problem.py:160-170,
 * pymde/average_distortion.py:32-33): one-time narrowing of the (p,2) int64 COO list to
 * int32, canonical orientation, sort by (attractive|repulsive, lhs, rhs), permuted
 * parameters.  `edges` is read, never written.  `p_total` is the divisor of the mean
 * (global edge count when `edges` is one shard of a larger problem; pass p otherwise).
 * Blocking (synchronises `stream` once to size the sort workspace).
 * ------------------------------------------------------------------------------------- */
int mde_edges_create(mde_edges_t** out, const int64_t* edges, int64_t p, int64_t n_items,
                     const float* par0, const float* par1 /* nullable */, const mde_fn_t* fn,
                     int64_t p_total, void* stream);
/* Same, with the embedding dimension: for embedding_dim <= 4 dense graphs (>= 64 edges per item) get a tile-resident
 * layout next to the sorted-SoA arrays -- the ELL pull records of pymde_b200/csrc/mde_ell.cu (one lane per owner: vertex
 * tiles of X live in shared memory, the records are streamed by TMA, built on the device), or the flat pull records of
 * mde_pull.cu when the ELL builder refuses the shape (more than 32 vertex tiles); everything else keeps the sorted-SoA
 * layout alone. */
int mde_edges_create_ex(mde_edges_t** out, const int64_t* edges, int64_t p, int64_t n_items,
                        const float* par0, const float* par1 /* nullable */, const mde_fn_t* fn,
                        int64_t p_total, int embedding_dim, void* stream);
int mde_edges_destroy(mde_edges_t* e);
int64_t mde_edges_count(const mde_edges_t* e);
/* which layout / kernel family the library chose: 0 = sorted SoA (quad / strided / wide kernels), 1 = tile records
 * (push kernel, shared-memory dst tile), 2 = pull records (directed entries, no shared-memory atomics), 3 = sorted SoA
 * + ELL pull records (one lane per owner, pymde_b200/csrc/mde_ell.cu: the fused evaluation runs on the ELL kernel,
 * value-only / per-edge outputs / external coefficients on the SoA kernels).
 * MDE_B200_LAYOUT=soa|tiles|pull|ell overrides the choice (A/B measurements). */
int mde_edges_kind(const mde_edges_t* e);
/* 1 when the layout was created with MDE_B200_DETERMINISTIC=1 and 1 <= embedding_dim <= 512: value AND gradient of
 * fused and external-coefficient evaluations at that m are bit-reproducible run to run and independent of scheduling
 * -- the reference's scatter_add_ is not (pymde/average_distortion.py:75-76).
 *   m <= 4: gradient contributions are accumulated as 64-bit fixed point (2^-40 resolution); two 64-bit reds per row
 *           update instead of one vector red.
 *   5 <= m <= 512: owner-complete rows -- every node's directed entries are evaluated by one group of lanes in a fixed
 *           order and its row is written once, with no atomics (lists longer than 256 entries in segments added in
 *           order); two row gathers per edge instead of one plus a row of reds. */
int mde_edges_deterministic(const mde_edges_t* e);
/* bytes of device memory held by the layout */
int64_t mde_edges_nbytes(const mde_edges_t* e);

/* The ELL pull records (layout kind 3) are built on the host; this is the same builder on HOST arrays, exported so the
 * CPU tests can decode the records and check the pull sums against the oracle without a device.  src / dst: p canonical
 * int32 edges, par0: weights; tile_rows_log2 = 0 and max_cta = 0 pick the defaults.  Buffers are malloc'ed, release them
 * with mde_ell_host_free.  Record format: pymde_b200/csrc/mde_ell.cu. */
typedef struct mde_ell_host {
  unsigned char* rec;  /* rec_bytes */
  uint32_t* rec_off;   /* [nrec + 1], units of 16 bytes */
  int32_t* bkt_tile;   /* [nbkt] neighbour tile of bucket b */
  int32_t* bkt_wt0;    /* [nbkt + 1] first record of bucket b */
  int32_t* cta_wt0;    /* [ncta + 1] record range of CTA c */
  int32_t* cta_bkt0;   /* [ncta] bucket holding cta_wt0[c] */
  int64_t rec_bytes, nrec, nslots, nentries, npadded;
  int32_t nbkt, ncta, tile_rows_log2, reserved;
} mde_ell_host_t;
int mde_ell_host_layout(int64_t n_items, int64_t p, int embedding_dim, const int32_t* src, const int32_t* dst,
                        const float* par0, int push_pull, int tile_rows_log2, int max_cta, mde_ell_host_t* out);
/* The builder the library itself uses: same layout, bit for bit, from DEVICE arrays (radix sorts + scans + one fill
 * kernel); the result is copied back into host buffers (GPU tests compare it with mde_ell_host_layout). */
int mde_ell_device_layout(int64_t n_items, int64_t p, int embedding_dim, const int32_t* src, const int32_t* dst,
                          const float* par0, int push_pull, int tile_rows_log2, int max_cta, mde_ell_host_t* out,
                          void* stream);
void mde_ell_host_free(mde_ell_host_t* h);

/* ---------------------------------------------------------------------------------------
 * Fused average distortion: value and gradient in ONE launch.
 * Replaces _AverageDistortion.forward + .backward (pymde/average_distortion.py:38-80) and
 * the penalty/loss modules it back-propagates through.
 *   loss_sum[0] += sum_k f_k(d_k)        (double, NOT divided by p; caller zeroes it; NULL skips
 *                  the one-block finalize and leaves per-block partials inside the layout)
 *   grad        += dE/dX contribution of this shard, already scaled by 1/p_total
 *                  (caller zeroes it; pass NULL for the forward-only branch, :64-65)
 * ------------------------------------------------------------------------------------- */
int mde_distortion(const mde_edges_t* e, const float* X, int m, float* grad /* nullable */,
                   double* loss_sum, void* stream);

/* Per-edge outputs in the CALLER'S edge order.  Replaces MDE.distances / MDE.distortions
 * (pymde/problem.py:252-307).  Either output may be NULL. */
int mde_edge_outputs(const mde_edges_t* e, const float* X, int m, float* distances,
                     float* distortions, void* stream);

/* Elementwise f_k(d_k) and f'_k(d_k) on caller-ordered arrays.  Replaces Function.forward of the
 * penalty / loss modules (pymde/functions/penalties.py:112-400, losses.py:61-239) and the autograd
 * pass through them (average_distortion.py:47-53).  par0 may have 1 element (broadcast) when
 * par0_len == 1.  Either output may be NULL. */
int mde_function_eval(const mde_fn_t* fn, const float* par0, int64_t par0_len, const float* par1,
                      const float* distances, int64_t p, float* f, float* fprime, void* stream);

/* Gradient scatter with caller-supplied per-edge coefficients g_k (caller's edge order):
 * grad += sum_k g_k (x_i - x_j)(e_i - e_j).  The backward of average_distortion.py:69-80
 * for distortion functions that are arbitrary Python callables (MDE_FN_EXTERNAL). */
int mde_scatter_external(const mde_edges_t* e, const float* X, int m, const float* g,
                         float* grad, void* stream);

/* ---------------------------------------------------------------------------------------
 * Constraint projections (pymde/constraints.py).  `ws` is a caller-provided device
 * workspace of at least mde_project_ws_bytes(n, m) bytes.
 * ------------------------------------------------------------------------------------- */
int64_t mde_project_ws_bytes(int64_t n, int m);
/* _Centered.project_onto_constraint, constraints.py:106-111: X -= column mean. */
int mde_project_centered(float* X, int64_t n, int m, void* ws, void* stream);
/* _Standardized.project_onto_constraint, constraints.py:194-195 -> util.py:129-171:
 * de-mean, then sqrt(n) * polar factor, computed as X (X^T X)^(-1/2) via the m x m Gram: a Jacobi eigensolver in
 * one warp for m <= 32, a tiled Gram kernel + fp64 Newton-Schulz inverse square root for 32 < m <= 256 (the reference
 * pins m = 250 in pymde/test_util.py:20-71).  m > 256: MDE_E_UNSUPPORTED.  The Gram is taken of X - s, s near the column
 * means (from the first 32 rows), so columns far from the origin keep their digits.  Asynchronous; a singular Gram is not an error code but a status word in
 * `ws`, read by mde_project_status.  The device solver's own retractions do not read it. */
int mde_project_standardized(float* X, int64_t n, int m, void* ws, void* stream);
/* Blocking: waits for `stream`, then stores in *status the status word of the last mde_project_standardized on `ws`
 * with this m: 0 ok, 1 when the de-meaned X is numerically rank deficient (n <= m, a constant or duplicated column,
 * smallest Gram eigenvalue <= 1e-12 x the largest for m <= 32, or a Newton-Schulz chain that did not converge for
 * m > 32; W and X are then not meaningful).  Returns 0 or an error code. */
int mde_project_status(const void* ws, int m, int* status, void* stream);
/* _Standardized.project_onto_tangent_space, constraints.py:186-192: Z -= (1/n) X (Z^T X).  m <= 256. */
int mde_tangent_standardized(const float* X, float* Z, int64_t n, int m, void* ws, void* stream);

/* ---------------------------------------------------------------------------------------
 * Device-resident projected L-BFGS.  Replaces optim.lbfgs (pymde/optim.py:69-184) driving
 * LBFGS.step (pymde/lbfgs.py:390-590) and _strong_wolfe (pymde/lbfgs.py:44-253).
 * All vectors, the quasi-Newton history, the Wolfe bracket and the per-iteration
 * statistics live on the device; the host enqueues work and reads back a status word.
 * ------------------------------------------------------------------------------------- */
typedef struct mde_solver_opts {
  int32_t constraint;       /* MDE_CONSTRAINT_* */
  int32_t memory_size;      /* L-BFGS history (optim.py:110) */
  int32_t max_iter;         /* capacity of the statistics arrays */
  int32_t mode;             /* must be 2: flat CUDA graphs of gated "steps" (one closure evaluation each), no
                               conditional nodes.  0 and 1 (retired drivers) give MDE_E_UNSUPPORTED, any other
                               value MDE_E_INVALID. */
  int64_t n_anchors;        /* MDE_CONSTRAINT_ANCHORED */
  const int64_t* anchors;   /* device (n_anchors,) */
  const float* anchor_values; /* device (n_anchors, m) */
  int32_t world_size;       /* >1: gradient/loss of each evaluation are summed across ranks */
  int32_t reserved;
} mde_solver_opts_t;

int mde_solver_create(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m,
                      const mde_solver_opts_t* opts, void* stream);
int mde_solver_destroy(mde_solver_t* s);
/* Start a solve from X0 (device, (n,m)); copies it (MDE.embed clones, problem.py:448-449). */
int mde_solver_begin(mde_solver_t* s, const float* X0, double eps, void* stream);
/* Same, with this solve's iteration cap (1 <= max_iter <= opts.max_iter of mde_solver_create, which sizes the
 * statistics buffers): one solver object serves embed() calls with different `max_iter`. */
int mde_solver_begin_ex(mde_solver_t* s, const float* X0, double eps, int max_iter, void* stream);
/* Run up to `iters` further iterations; stops early on convergence (||grad||_F <= eps,
 * optim.py:165).  Blocking.  On return *iters_done = total iterations so far,
 * *converged = 1 if the residual test fired.  Returns MDE_E_NAN where the reference raises
 * SolverError. */
int mde_solver_run(mde_solver_t* s, int iters, int* iters_done, int* converged, void* stream);

/* Diagnostics: %globaltimer stamps (ns) of the last step that started an iteration:
 * [0] entry of the head kernel's last block, [1] its scalar stage begins, [2] solver state staged in shared memory,
 * [3] partials reduced, [4] previous step finished / phase chosen, [5] history update + two-loop done,
 * [6] before the state is written back, [7] first block of the vector kernel that follows.  No reference counterpart. */
int mde_solver_debug_times(mde_solver_t* s, unsigned long long* out8, void* stream);
/* Diagnostics: the L-BFGS state of a solve paused between two mde_solver_run calls, copied to host buffers (blocking;
 * MDE_E_INVALID when the solve is not paused).  g: (n*m) gradient of the last evaluation; g_prev, d: (n*m) gradient
 * and direction of the last completed iteration; S, Y: (memory_size, n*m) receive the *count stored pairs in logical
 * order, oldest first; *h_diag, *n_iter: the scaling of the two-loop recursion and the iterations since the last
 * reset.  Changes no device state.  No reference counterpart. */
int mde_solver_debug_lbfgs(mde_solver_t* s, float* g, float* g_prev, float* d, float* S, float* Y, int* count,
                           double* h_diag, int* n_iter, void* stream);
/* Device pointer to the current iterate (n,m). */
float* mde_solver_x(mde_solver_t* s);
/* Copy statistics to host arrays of length >= iterations done (blocking):
 * average_distortions, residual_norms, step_size_percents (optim.py:30-47), step lengths. */
int mde_solver_stats(mde_solver_t* s, double* average_distortions_host, double* residual_norms_host,
                     double* step_size_percents_host, double* step_lengths_host, int64_t* func_evals_host,
                     void* stream);

/* Distortion functions that are arbitrary callables (pymde/problem.py:36-193 accepts any (p,) -> (p,) torch function):
 * the solver runs the caller's part of every evaluation between two of its own gated kernels,
 *     distances d (caller's edge order) -> caller: fpp, loss -> g_k = fpp_k / d_k (non-finite g -> 1) -> gradient scatter
 * where fpp = d mean_k f(d_k) / d d (fp32) and loss = sum_k f(d_k) (one fp64 value); the loss takes the route of a
 * built-in loss (a non-finite one ends in MDE_E_NAN where the reference raises SolverError).  The caller's part is
 * given in one of two forms:
 *   graph  a cudaGraph_t (as void*) that reads d and writes fpp and loss, with kernel, memset and memcpy nodes only
 *          (anything else: MDE_E_UNSUPPORTED).  It is added as a child node to every step of the solver's CUDA graphs
 *          and, unlike the solver's kernels, it is not gated: in the surplus steps after the device paused it runs
 *          again on a stale d, and nothing reads its result.  The graph is copied; its buffers must outlive the solver.
 *   hook   fn(user, d, fpp, loss, stream), called on the host at every evaluation, must enqueue the same work on
 *          `stream` and return 0 (non-zero is returned by mde_solver_run).  Steps are then stream-launched.
 * Exactly one of `graph` and `fn` is set.  d and fpp hold mde_edges_count(e) floats. */
typedef int (*mde_external_fn)(void* user, const float* d, float* fpp, double* loss, void* stream);
typedef struct mde_external {
  float* d;             /* written by the solver, read by the caller's part */
  float* fpp;           /* written by the caller's part, read by the solver */
  double* loss;         /* written by the caller's part, read by the solver */
  void* graph;          /* cudaGraph_t, or NULL */
  mde_external_fn fn;   /* or NULL */
  void* user;
} mde_external_t;
/* One GPU only (opts->world_size == 1). */
int mde_solver_create_external(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m,
                               const mde_solver_opts_t* opts, const mde_external_t* ext, void* stream);
/* Replace the caller's part of a solver made by mde_solver_create_external and rebuild its step graphs (a callable
 * captured anew).  Blocking. */
int mde_solver_set_external(mde_solver_t* s, const mde_external_t* ext, void* stream);

/* Constraints whose projections the caller defines (pymde/constraints.py:7-91, any Constraint subclass), on the
 * device solver (opts->constraint == MDE_CONSTRAINT_CUSTOM).  The caller's projections run on its own staging
 * buffers, never in place on the solver's iterate X or gradient g:
 *     retraction  [X -> u] -> caller: retract(u) in place -> [u -> X]      after the iterate moved
 *     tangent     [X -> xt, g -> gt] -> caller: tangent(xt, gt), gt in place -> [gt -> g]   after every evaluation
 * The bracketed copies are gated like the solver's own kernels (a step at the current iterate does not retract;
 * the retraction of an accepted earlier trial does not evaluate); the caller's part is not gated, so in the steps
 * after the device paused it runs again on stale staging buffers and nothing reads its result.  A projection that
 * yields non-finite values ends, through the loss, in MDE_E_NAN.  The caller's part is given either as two CUDA graphs
 * (kernel, memset and memcpy nodes only, else MDE_E_UNSUPPORTED; added as child nodes to every step), or as a hook
 * fn(user, which, stream), which = 0 retraction / 1 tangent, that enqueues the same work on `stream` and returns 0
 * (non-zero is returned by mde_solver_run).  Either both graphs or fn are set.  u, xt and gt each hold at least
 * npad = ceil(n*m / 32) * 32 floats, 16-byte aligned, rows of m floats from the start; they must outlive the solver
 * (or the next mde_solver_set_constraint_part). */
typedef int (*mde_constraint_fn)(void* user, int which /* 0 retract, 1 tangent */, void* stream);
typedef struct mde_constraint_part {
  float* u;             /* retraction: iterate in, retracted iterate out */
  float* xt;            /* tangent projection: the iterate */
  float* gt;            /* tangent projection: gradient in, projected gradient out */
  void* retract_graph;  /* cudaGraph_t, or NULL */
  void* tangent_graph;  /* cudaGraph_t, or NULL */
  mde_constraint_fn fn; /* or NULL */
  void* user;
} mde_constraint_part_t;
/* One GPU only (opts->world_size == 1, else MDE_E_INVALID).  `ext` is a callable distortion function as for
 * mde_solver_create_external, or NULL for the layout's table function.  When any caller's part is a hook, the steps are
 * stream-launched, and the caller's parts given as graphs are launched inside them. */
int mde_solver_create_custom(mde_solver_t** out, const mde_edges_t* e, int64_t n, int m,
                             const mde_solver_opts_t* opts, const mde_external_t* ext,
                             const mde_constraint_part_t* part, void* stream);
/* Replace the constraint part of a solver made by mde_solver_create_custom and rebuild its step graphs.  Blocking. */
int mde_solver_set_constraint_part(mde_solver_t* s, const mde_constraint_part_t* part, void* stream);

/* Multi-GPU hook (world_size > 1): after every distortion launch the solver calls
 * `fn(user, buf, count, stream)` which must sum the float32 buffer in place across ranks
 * on `stream` (an NCCL all-reduce).  buf = [partial gradient (n*m) | loss hi | loss lo]. */
typedef int (*mde_allreduce_fn)(void* user, float* buf, int64_t count, void* stream);
int mde_solver_set_allreduce(mde_solver_t* s, mde_allreduce_fn fn, void* user);

/* Peer-memory all-reduce (world_size > 1, one process per GPU on one NVLink node): the preferred path.
 * Every rank exports the cudaIpc handle of its partial-gradient region (64 bytes), the ranks exchange the handles
 * out of band (torch.distributed.all_gather in pymde_b200/dist.py), and mde_solver_comm_connect maps the peers'
 * regions.  From then on each evaluation's all-reduce is done by the library's own kernels over NVLink
 * (flag handshake + rank-ordered sums: bit-identical on every rank), graph-captured with the rest of the step;
 * the host hook above is not used.  `handles` = world_size handles, `handle_stride` bytes apart, rank order. */
#define MDE_IPC_HANDLE_BYTES 64
int mde_solver_comm_export(mde_solver_t* s, void* handle_out, int64_t handle_bytes);
int mde_solver_comm_connect(mde_solver_t* s, int rank, const void* handles, int64_t handle_stride, void* stream);

/* ---------------------------------------------------------------------------------------
 * Problem construction next to the path (SURVEY section 8 row f3): exact k-nearest neighbours.
 * Replaces the neighbour search of pymde/preprocess/data_matrix.py:91-178 (k_nearest_neighbors: scikit-learn brute
 * force below 10 000 rows, the approximate pynndescent above; a third-party dependency either way).  X is a device
 * row-major n x d fp32 matrix.  For every row i the k rows nearest to it in Euclidean distance (i itself excluded)
 * are written to idx_out[i*k .. i*k+k) in ascending distance with their exact fp32 SQUARED distances in d2_out.
 * Cross terms run on the tensor cores (wgmma, bf16 hi/lo split, fp32 accumulate in registers) with a running
 * top-32 per row; the 32 candidates are re-ranked with exact fp32 distances, so the result is that of a brute-force
 * fp32 search (equal-distance ties aside).  1 <= k <= mde_knn_max_k() (24), k <= n - 1.  `ws`: 1024-byte aligned
 * device scratch of mde_knn_ws_bytes(n, d) bytes.  Asynchronous on `stream`. */
int mde_knn_max_k(void);
int mde_knn_ws_bytes(int64_t n, int d, size_t* bytes);
int mde_knn(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
            void* stream);

/* The same search on a sparse data matrix, without densifying it (pymde/preprocess/data_matrix.py:19,99 accepts
 * scipy.sparse input).  Device CSR of an n x d matrix: int64 indptr[n+1] (indptr[0] = 0, indptr[n] = nnz), int32
 * indices[nnz] strictly increasing within a row and below d, fp32 values[nnz]; nnz may exceed 2^31.  Output contract
 * of mde_knn, except that the distances are the exact squared distances summed in fp64 and rounded once to fp32, and
 * the k rows are the k smallest (distance, index) pairs in lexicographic order: the result is fully determined,
 * ties included.  Cross terms run on the tensor cores over the 64-feature blocks both tiles occupy (features ordered
 * by descending document frequency); nothing n x d sized is allocated.  1 <= k <= mde_knn_max_k() (24),
 * k <= n - 1.  `ws`: 1024-byte aligned device scratch of mde_knn_csr_ws_bytes(n, d, nnz) bytes (about 20 bytes per
 * non-zero and 260 per row, plus 20 per feature and the sort's scratch).  MDE_E_INVALID also when the CSR is malformed (checked on the device).
 * Blocking (one status read after the check). */
int mde_knn_csr_ws_bytes(int64_t n, int d, int64_t nnz, size_t* bytes);
int mde_knn_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d, int64_t nnz,
                int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream);
/* The same two searches for 1 <= k <= mde_knn_wide_max_k() (64), k <= n - 1: arguments, output contract, tie rules
 * and return codes of mde_knn and mde_knn_csr (the CSR check included).  A running top-96 per row, kept in shared
 * memory, feeds the exact re-rank.  For k <= 24 the result is that of mde_knn / mde_knn_csr, which remain the faster
 * searches there.  `ws`: 1024-byte aligned device scratch of mde_knn_wide_ws_bytes(n, d) or
 * mde_knn_csr_wide_ws_bytes(n, d, nnz) bytes (256 more bytes per row than the narrow searches).  mde_knn_wide is
 * asynchronous on `stream`, mde_knn_csr_wide blocking as mde_knn_csr. */
int mde_knn_wide_max_k(void);
int mde_knn_wide_ws_bytes(int64_t n, int d, size_t* bytes);
int mde_knn_wide(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws,
                 size_t ws_bytes, void* stream);
int mde_knn_csr_wide_ws_bytes(int64_t n, int d, int64_t nnz, size_t* bytes);
int mde_knn_csr_wide(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                     int64_t nnz, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes, void* stream);
/* APPROXIMATE k-nearest neighbours of a dense matrix by NN-descent, for n too large for the exact O(n^2 d) search.
 * Output contract of mde_knn with "the k nearest rows" replaced by "k rows found by the search": k distinct rows per
 * row, never the row itself, ascending by (squared distance, index), with the exact fp32 squared distances of the
 * re-rank of mde_knn / mde_knn_wide (a pair found by both searches carries the same bits).  1 <= k <=
 * mde_knn_approx_max_k() (64), k <= n - 1.  The result is a function of (X, k, seed) alone: identical bits from run
 * to run, whatever the workspace held.  When n - 1 <= 32 (k <= 24) or n - 1 <= 96 (k > 24) every row's list holds
 * every other row and the result is that of the exact search.  `ws`: 1024-byte aligned device scratch of
 * mde_knn_approx_ws_bytes(n, d, k) bytes (about 1.1 KB per row for k <= 24, 1.9 KB for k > 24).  Return codes of
 * mde_knn_wide (MDE_E_UNSUPPORTED for n >= 2^31 - 128).  Blocking: one 8-byte read per iteration.
 * mde_knn_approx_ex also writes the number of NN-descent iterations to *iterations (nullable). */
int mde_knn_approx_max_k(void);
int mde_knn_approx_ws_bytes(int64_t n, int d, int k, size_t* bytes);
int mde_knn_approx(const float* X, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws,
                   size_t ws_bytes, void* stream);
int mde_knn_approx_ex(const float* X, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out, float* d2_out,
                      void* ws, size_t ws_bytes, void* stream, int* iterations);
/* The same NN-descent search on a sparse data matrix, without densifying it.  Input contract of mde_knn_csr (the
 * device CSR check included: MDE_E_INVALID when malformed); output contract of mde_knn_approx, with the distances of
 * mde_knn_csr / mde_knn_csr_wide: the exact squared distance summed in fp64 and rounded once to fp32, which is also
 * the distance the search itself compares, so a pair found by the exact and the approximate sparse search carries the
 * same bits.  The result is a function of (CSR, k, seed) alone, whatever the workspace held.  When n - 1 <= 32
 * (k <= 24) or n - 1 <= 96 (k > 24) the result is that of mde_knn_csr / mde_knn_csr_wide, ties included.
 * 1 <= k <= mde_knn_approx_max_k() (64), k <= n - 1; MDE_E_UNSUPPORTED for n >= 2^31 - 128.  `ws`: 1024-byte aligned
 * device scratch of mde_knn_approx_csr_ws_bytes(n, d, nnz, k) bytes: about 1.1 KB per row for k <= 24 (1.9 KB for
 * k > 24), 36 bytes per non-zero and 20 per feature, plus 8 MB (a host-computed bound on the sort's scratch; the call
 * returns MDE_E_ALLOC should the sort need more).  Blocking: the CSR check and one 8-byte read per iteration.
 * mde_knn_approx_csr_ex also writes the number of NN-descent iterations to *iterations (nullable). */
int mde_knn_approx_csr_ws_bytes(int64_t n, int d, int64_t nnz, int k, size_t* bytes);
int mde_knn_approx_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                       int64_t nnz, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
                       void* stream);
int mde_knn_approx_csr_ex(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                          int64_t nnz, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws,
                          size_t ws_bytes, void* stream, int* iterations);
/* Euclidean distances ||x_a - x_b|| of p row pairs (device int64 pairs[p][2]) of the same CSR, into out[p] (fp32):
 * a sorted merge of the two rows summed in fp64, sqrt in fp64, one rounding (pymde/preprocess/data_matrix.py:59-70
 * takes the norm of the difference in scipy).  MDE_E_INVALID for a malformed CSR or a pair index outside [0, n).
 * Blocking. */
int mde_pair_dist_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                      const int64_t* pairs, int64_t p, float* out, void* stream);
/* Neighbour lists to a weighted undirected edge list (replaces pymde/preprocess/data_matrix.py:172-178 and
 * graph.py:75-110: Graph.from_edges of the directed pairs, then .edges / .weights).  idx: device int32 [n][k],
 * row-major, as mde_knn*, mde_knn_approx* and mde_graph_knn write it; -1 means "no entry" and may sit anywhere in a
 * row.  The output is every unordered pair {i, j} with at least one entry i -> j or j -> i, as int64 rows (i, j) with
 * i < j sorted by (i, j), with the fp32 weight (number of entries i -> j) + (number of entries j -> i): 1 or 2 for the
 * searches, and duplicates inside a row are counted too.  Two calls on one workspace: mde_knn_graph_count checks the
 * entries and counts the pairs (*count); mde_knn_graph_emit then writes edges_out[count][2] and weights_out[count]
 * from what the count left in `ws` (same n, k and ws; the call is skipped when count is 0).  An entry equal to its
 * own row or outside [-1, n) gives MDE_E_INVALID (checked on the device).  No atomics order the output: the result
 * is a function of (idx, n, k) alone, whatever the workspace held, and a row listed by every other row costs no more
 * than its entries.  1 <= k <= mde_knn_graph_max_k() (64), n >= 1; MDE_E_UNSUPPORTED for n k >= 2^31 - 1.  `ws`:
 * 1024-byte aligned device scratch of mde_knn_graph_ws_bytes(n, k) bytes (about 25 bytes per entry, plus 16 MB, a
 * host-computed bound on the sort's scratch; the count returns MDE_E_ALLOC should the sort need more).  The count is
 * blocking (one 8-byte read); the emit is asynchronous on `stream`. */
int mde_knn_graph_max_k(void);
int mde_knn_graph_ws_bytes(int64_t n, int k, size_t* bytes);
int mde_knn_graph_count(const int32_t* idx, int64_t n, int k, void* ws, size_t ws_bytes, int64_t* count,
                        void* stream);
int mde_knn_graph_emit(int64_t n, int k, const void* ws, size_t ws_bytes, int64_t* edges_out, float* weights_out,
                       void* stream);

/* ---------------------------------------------------------------------------------------
 * Problem construction next to the path (SURVEY section 8 row f4).
 * Hop-count shortest paths of an UNWEIGHTED undirected graph given as a symmetric CSR adjacency (device int32
 * indptr[n+1], indices[nnz]).  Replaces the one-BFS-per-node pool of pymde/preprocess/graph.py:310-474 and
 * pymde/preprocess/_graph.pyx:10-52: for every source s in [s_begin, s_end) and every node v > s reachable in
 * <= max_length hops (0 = unlimited), the triple (s, v, hops) is kept with probability `retain` (counter-based
 * hash of (seed, s, v)) and appended to out_src / out_dst / out_len (capacity `cap`, unsorted).  *count_dev
 * (device, caller zeroes it) receives the number of triples produced; if it exceeds `cap` the surplus was dropped
 * and the caller re-runs with larger buffers.  Blocking (one status read per BFS level).
 * `ws` >= mde_graph_hops_ws_bytes(n) bytes of device scratch. */
int64_t mde_graph_hops_ws_bytes(int64_t n);
int mde_graph_hops(const int32_t* indptr, const int32_t* indices, int64_t n, int64_t s_begin, int64_t s_end,
                   int max_length, double retain, uint64_t seed, int32_t* out_src, int32_t* out_dst,
                   float* out_len, int64_t cap, unsigned long long* count_dev, void* ws, int64_t ws_bytes,
                   void* stream);

/* Shortest paths of a WEIGHTED undirected graph (SURVEY section 8 row f4).  Replaces the chunked scipy Dijkstra of
 * pymde/preprocess/graph.py:345-474 (and its per-source helper, pymde/preprocess/graph.py:311-335).  Device CSR:
 * int32 indptr[n+1], indices[nnz], fp32 weights[nnz] (NULL = unit weights); both directions of every edge present,
 * entries positive and finite, duplicates allowed (the shorter wins).  Lengths are fp64 sums of the widened
 * weights, so they equal scipy's dijkstra bit for bit after the cast to fp32.  Same output contract as
 * mde_graph_hops: for every source s in [s_begin, s_end) and every node v > s with length <= max_length (<= 0 or
 * inf: unlimited), the triple (s, v, length) is kept when the same counter-based hash of (seed, s, v) falls under
 * `retain` (one seed selects the same pairs in both engines), appended unsorted to out_src / out_dst / out_len
 * (capacity `cap`); *count_dev (caller zeroes it) receives the total, and the caller re-runs with larger buffers
 * when it exceeds `cap`.  Sources run in batches of B (a multiple of 32), the largest that `ws_bytes` holds:
 * `ws` >= mde_graph_sssp_ws_bytes(n, 32) bytes of device scratch; mde_graph_sssp_ws_bytes(n, B) is the size for
 * batches of B (-1 if B is not a positive multiple of 32).  Per batch the work is proportional to the
 * (source, node) pairs the searches reach.  Blocking (one status read per few relaxation rounds, at most n
 * rounds per batch). */
int64_t mde_graph_sssp_ws_bytes(int64_t n, int batch);
int mde_graph_sssp(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n,
                   int64_t s_begin, int64_t s_end, double max_length, double retain, uint64_t seed, int32_t* out_src,
                   int32_t* out_dst, float* out_len, int64_t cap, unsigned long long* count_dev, void* ws,
                   int64_t ws_bytes, void* stream);

/* k nearest neighbours of every node under the shortest-path metric of the same CSR (weights NULL = unit).
 * Replaces pymde/preprocess/graph.py:503-586 (chunked Dijkstra with limit = max_distance, then a partition per
 * row).  For every node s, the k smallest (length, node index) pairs in lexicographic order, s itself excluded,
 * length <= max_distance (<= 0 or inf: unlimited), go to out_idx[s*k .. s*k+k) (int32) and out_len (fp32),
 * ascending; rows with fewer than k such nodes are padded with -1 / +inf.  Ties break by node index, so the result
 * is fully determined.  1 <= k <= mde_graph_knn_max_k() (64).  `ws` >= mde_graph_knn_ws_bytes(n, 32) bytes; the
 * batch is derived from `ws_bytes` as for mde_graph_sssp.  Blocking. */
int mde_graph_knn_max_k(void);
int64_t mde_graph_knn_ws_bytes(int64_t n, int batch);
int mde_graph_knn(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n, int k,
                  double max_distance, int32_t* out_idx, float* out_len, void* ws, int64_t ws_bytes, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MDE_B200_H */
