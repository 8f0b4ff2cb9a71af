// mde_knn_approx.cu -- approximate k-nearest neighbours of the rows of a dense data matrix by NN-descent (Dong,
// Moses and Li 2011, in the GPU form of GNND, Wang et al. 2021).  Opt-in next to the exact mde_knn / mde_knn_wide,
// whose cost grows as n^2 d: NN-descent costs about (iterations x n x 64 staged rows x d).
//
// Every row keeps a list of KB (distance, index) entries, KB = 32 for k <= 24 and 96 for k <= 64, as one sorted array
// of 64-bit keys ((fp32 distance bits << 32) | index; all ones = empty) and one "new" flag per entry.  An iteration is
//
//   sample   per row, the S new and S old list entries of lowest hash priority (seed, iteration, row, neighbour); the
//            sampled new entries become old, and every sample (u -> v) is offered to v's reverse reservoir
//   join     one CTA per row u: the union of its new and old, forward and reverse samples (<= 64 rows, deduplicated,
//            new first) is staged in shared memory 64 features at a time; every pair (a, b) with a new member gets
//            its squared distance on the CUDA cores and is offered to a and b when it beats the worst entry of the
//            target's list at the start of the iteration and is not in that list already
//   merge    per row, the list and the offers it received: duplicates dropped, the KB smallest keys kept, entries
//            that came from offers flagged new; the number of such entries is counted
//
// and the host stops when fewer than 0.001 n KB entries changed or after max(5, ceil(log2 n)) iterations.  The final
// lists go to the re-rank kernels of mde_knn (knn_rerank_kernel for 32 candidates, knn_wide_rerank_kernel for 96),
// so the output contract and the distance arithmetic are those of the exact search.  A 16-bit matrix (IEEE fp16 or
// bf16, mde_knn16_approx) or an 8-bit one (uint8 or int8, mde_knn8_approx) is read in place: DenseRows, the join and
// the re-rank take the element type as a template parameter and convert each element to fp32 as they load it, so
// every distance, and with it the whole search, has the bits of the fp32 search on X.float().
//
// Determinism.  Offers and reverse samples arrive in a racy order, so they are collected in cascade reservoirs: R
// 64-bit keys per row, all ones when empty; inserting x runs y = atomicMin(&r[i], x), x = max(x, y) down the slots.
// Slot i ends up with the i-th smallest key offered (with multiplicity) whatever the interleaving.  Every distance
// used inside the search is the sequential fp32 sum of fmaf((a_f - b_f)^2) over f = 0 .. d-1, a function of the
// unordered pair alone, so a pair offered twice carries the same key and duplicates are exact.  Everything the search
// reads is written by it first: nothing depends on the workspace's earlier contents.
//
// Sparse rows (mde_knn_approx_csr).  The CSR is validated and re-sorted by prepare_csr (mde_knn_sparse.cu: features
// by descending document frequency), and every distance of the search is merge_dist2 over those rows: the fp64 sum
// in column order rounded once to fp32, again a function of the unordered pair alone.  Only init and join depend on
// the row format (DenseRows, CsrRows); sample, merge, the reservoirs, the stop rule and the driver are shared.  The
// CSR join stages its candidates' (column, value) slices in shared memory while they fit kCsrStage entries and
// merges the others from global memory; one thread merges one pair.  The final lists go to knn_csr_rerank_kernel /
// knn_csr_wide_rerank_kernel, so a pair found by both sparse searches carries the same bits.
#include <cuda_runtime.h>

#include <cstdint>

#include "mde_common.cuh"
#include "mde_knn_csr.cuh"
#include "mde_knn_select.cuh"

using namespace mde;

namespace {

constexpr int kS = 16;                 // new and old samples per row and direction
constexpr int kCand = 4 * kS;          // join candidates: forward new, reverse new, forward old, reverse old
constexpr int kRes = 32;               // offer reservoir slots per row
constexpr int kNarrowMaxK = 24;        // k <= 24: lists of 32 and knn_rerank_kernel (as mde_knn); else 96
constexpr int kFC = 64;                // features per staged chunk in the join
constexpr int kJoinThreads = 128;
constexpr int kJoinTiles = 100;        // 4 x 4 pair tiles (ta < 8 <= 16 new rows, ta <= tb < 16)
constexpr int kDeltaInv = 1000;        // stop when fewer than n KB / 1000 entries changed
constexpr int kCsrJoinThreads = 256;
constexpr int kCsrStage = 5632;        // CSR join: staged (column, value) entries per CTA (44 KB)
constexpr unsigned long long kEmpty = ~0ull;
static_assert(kRes == 32 && 2 * kS == 32, "the reservoirs of a row are reset by one warp, one slot per lane");
static_assert(kCand == 64, "the join's pair tiles cover 16 groups of 4 candidates");

__device__ __forceinline__ uint64_t mix64(uint64_t x) {  // splitmix64 finaliser
  x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ull;
  x ^= x >> 27; x *= 0x94d049bb133111ebull;
  return x ^ (x >> 31);
}
__device__ __forceinline__ uint64_t hash4(uint64_t seed, uint64_t a, uint64_t b, uint64_t c) {
  return mix64(mix64(mix64(seed + 0x9e3779b97f4a7c15ull * (a + 1)) ^ b) + c);
}

// The one distance of the search: sequential fp32 sum over the features (the join's tiles add in the same order).
template <class T>
__device__ __forceinline__ float seq_dist(const T* __restrict__ a, const T* __restrict__ b, int d) {
  float acc = 0.0f;
  for (int f = 0; f < d; ++f) { const float t = elem_f32(a[f]) - elem_f32(b[f]); acc = fmaf(t, t, acc); }
  return acc;
}

__device__ __forceinline__ unsigned long long make_key(float dist, uint32_t idx) {
  return ((unsigned long long)__float_as_uint(dist) << 32) | idx;
}

// Cascade insertion into a reservoir of R ascending slots.  Both shortcuts are exact: a slot only ever decreases, so
// a read r[i] <= x means the atomic would return <= x and change nothing, and x > r[R-1] (strict: an equal key must
// still take its slot) means x is not among the R smallest.
__device__ __forceinline__ void reservoir_insert(unsigned long long* r, int R, unsigned long long x) {
  if (x > __ldcg(r + R - 1)) return;
  for (int i = 0; i < R; ++i) {
    if (__ldcg(r + i) <= x) continue;
    const unsigned long long y = atomicMin(r + i, x);
    x = x > y ? x : y;
    if (x == kEmpty) return;
  }
}

// Whether key x is in a row's sorted list.  The lists are not written during the join, so the read is stable, and a
// pair's key depends on the pair alone, so key equality is index equality.
template <int KB>
__device__ __forceinline__ bool in_list(const unsigned long long* __restrict__ l, unsigned long long x) {
  int lo = 0, hi = KB;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(l + mid) < x) lo = mid + 1; else hi = mid; }
  return lo < KB && __ldg(l + lo) == x;
}

// The row formats: the one distance of the search between rows a and b.  T: the element type of a dense matrix.
template <class T>
struct DenseRows {
  const T* X;
  int d;
  __device__ __forceinline__ float dist(int64_t a, int64_t b) const { return seq_dist(X + a * d, X + b * d, d); }
};
struct CsrRows {  // the rows as prepare_csr re-sorts them
  const int64_t* indptr;
  const int32_t* cols;
  const float* vals;
  __device__ __forceinline__ float dist(int64_t a, int64_t b) const { return (float)merge_dist2(indptr, cols, vals, a, b); }
};

__device__ __forceinline__ unsigned long long gcd_u64(unsigned long long a, unsigned long long b) {
  while (b) { const unsigned long long t = a % b; a = b; b = t; }
  return a;
}

// ---------------------------------------------------------------------------------------------------------------
// init: one warp per row.  The list starts with min(KB, n - 1) distinct rows: all others when n - 1 <= KB, else the
// rows u + 1 + (a + j b) mod (n - 1) for slots j, with a and b (coprime to n - 1) hashed from (seed, u).  Resets the
// row's reservoirs.
// ---------------------------------------------------------------------------------------------------------------
template <int KB, class Rows>
__global__ void __launch_bounds__(256)
nnd_init_kernel(Rows rows, int64_t n, uint64_t seed, unsigned long long* __restrict__ keys,
                uint8_t* __restrict__ flags, uint32_t* __restrict__ thr, unsigned long long* __restrict__ offers,
                unsigned long long* __restrict__ rev) {
  __shared__ unsigned long long s_k[8][KB];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t row = (int64_t)blockIdx.x * 8 + w;
  if (row >= n) return;
  const unsigned long long m = (unsigned long long)(n - 1);
  unsigned long long a = 0, b = 1;
  if (m > (unsigned long long)KB) {
    a = hash4(seed, 0, (uint64_t)row, 0) % m;
    b = 1 + hash4(seed, 1, (uint64_t)row, 0) % (m - 1);
    while (gcd_u64(b, m) != 1) b = (b + 1 < m) ? b + 1 : 1;
  }
#pragma unroll 1  // one distance at a time: unrolled, the CSR merges spill
  for (int s = 0; s < KB / 32; ++s) {
    const int j = lane + 32 * s;
    unsigned long long key = kEmpty;
    if ((unsigned long long)j < m) {
      const unsigned long long off = (m > (unsigned long long)KB) ? 1 + (a + (unsigned long long)j * b) % m : 1 + j;
      const int64_t c = (int64_t)(((unsigned long long)row + off) % (unsigned long long)n);
      key = make_key(rows.dist(row, c), (uint32_t)c);
    }
    s_k[w][j] = key;
  }
  __syncwarp();
#pragma unroll
  for (int s = 0; s < KB / 32; ++s) {
    const int j = lane + 32 * s;
    const unsigned long long key = s_k[w][j];
    int rank = 0;  // keys are distinct except the empty ones, which keep their slot order
    for (int q = 0; q < KB; ++q) {
      const unsigned long long o = s_k[w][q];
      rank += (o < key) || (o == key && q < j);
    }
    keys[row * KB + rank] = key;
    flags[row * KB + rank] = key != kEmpty;
    if (rank == KB - 1) thr[row] = (uint32_t)(key >> 32);
  }
  offers[row * kRes + lane] = kEmpty;
  rev[row * 2 * kS + lane] = kEmpty;
}

// ---------------------------------------------------------------------------------------------------------------
// sample: one warp per row.  fwd[u] = S new then S old list entries (-1 padded) of lowest priority; the sampled new
// entries are flagged old; each sample u -> v goes to v's reverse reservoir (new: rev[v][0, S), old: [S, 2S)) with
// the key (priority << 32 | u).
// ---------------------------------------------------------------------------------------------------------------
template <int KB>
__global__ void __launch_bounds__(256)
nnd_sample_kernel(int64_t n, uint64_t seed, int iter, const unsigned long long* __restrict__ keys,
                  uint8_t* __restrict__ flags, int32_t* __restrict__ fwd, unsigned long long* __restrict__ rev) {
  __shared__ unsigned long long s_p[8][KB];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t row = (int64_t)blockIdx.x * 8 + w;
  if (row >= n) return;
  constexpr int P = KB / 32;
  unsigned long long sk[P];
  int n_new = 0, n_old = 0;
#pragma unroll
  for (int s = 0; s < P; ++s) {
    const int j = lane + 32 * s;
    const unsigned long long key = keys[row * KB + j];
    const bool valid = key != kEmpty, is_new = valid && flags[row * KB + j];
    const uint32_t idx = (uint32_t)key;
    const uint32_t pr = (uint32_t)(hash4(seed, 2 + (uint64_t)iter, (uint64_t)row, idx) >> 33);  // 31 bits
    // new entries order before old ones, each by (priority, index)
    sk[s] = valid ? ((unsigned long long)!is_new << 63) | ((unsigned long long)pr << 32) | idx : kEmpty;
    s_p[w][j] = sk[s];
    n_new += __popc(__ballot_sync(kFull, is_new));
    n_old += __popc(__ballot_sync(kFull, valid && !is_new));
  }
  __syncwarp();
  int32_t* f = fwd + row * 2 * kS;
#pragma unroll
  for (int s = 0; s < P; ++s) {
    if (sk[s] == kEmpty) continue;
    int rank = 0;
    for (int q = 0; q < KB; ++q) rank += s_p[w][q] < sk[s];
    const bool is_new = !(sk[s] >> 63);
    const int r = is_new ? rank : rank - n_new;
    if (r >= kS) continue;
    const uint32_t idx = (uint32_t)sk[s];
    const unsigned long long rk = (sk[s] & 0x7fffffff00000000ull) | (uint64_t)row;
    f[(is_new ? 0 : kS) + r] = (int32_t)idx;
    if (is_new) flags[row * KB + lane + 32 * s] = 0;
    reservoir_insert(rev + (int64_t)idx * 2 * kS + (is_new ? 0 : kS), kS, rk);
  }
  if (lane < kS) {
    if (lane >= n_new) f[lane] = -1;
  } else {
    if (lane - kS >= n_old) f[lane] = -1;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// join, shared by both row formats.  Candidates of row u: forward new, reverse new (slots 0..31 after compaction),
// forward old, reverse old (slots 32..63), each row once (its first, i.e. newest, occurrence); s_cnt = (new, old)
// counts.  Resets u's reverse reservoirs.  Called by every thread of the CTA (>= 64 threads).
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void join_candidates(int64_t u, const int32_t* __restrict__ fwd,
                                                unsigned long long* __restrict__ rev, const uint32_t* __restrict__ thr,
                                                int* s_raw, int* s_idx, uint32_t* s_thr, int* s_cnt) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  if (t < kCand) {
    const int grp = t / kS, q = t % kS;  // 0 fwd new, 1 rev new, 2 fwd old, 3 rev old
    int c;
    if (grp == 0 || grp == 2) {
      c = fwd[u * 2 * kS + (grp == 0 ? 0 : kS) + q];
    } else {
      unsigned long long* slot = rev + u * 2 * kS + (grp == 1 ? 0 : kS) + q;
      const unsigned long long key = *slot;
      *slot = kEmpty;
      c = key == kEmpty ? -1 : (int)(uint32_t)key;
    }
    s_raw[t] = c;
  }
  __syncthreads();
  if (t < kCand) {  // warps 0 (new) and 1 (old), whole
    const int c = s_raw[t];
    bool valid = c >= 0;
    for (int q = 0; q < t; ++q) valid &= s_raw[q] != c;
    const unsigned mask = __ballot_sync(kFull, valid);
    if (valid) {
      const int p = warp * 32 + __popc(mask & ((1u << lane) - 1));
      s_idx[p] = c;
      s_thr[p] = thr[c];
    }
    if (lane == 0) s_cnt[warp] = __popc(mask);
  }
  __syncthreads();
}

// The pair (a, b) of candidate slots at distance bits db, offered to both rows: when it beats the worst entry of the
// target's list at the start of the iteration and is not in that list already.  An offer that is already in the list
// is dropped before it can take a reservoir slot: the closest pairs are offered again and again, and would otherwise
// crowd the genuinely new candidates out of the reservoir.
template <int KB>
__device__ __forceinline__ void offer_pair(const unsigned long long* __restrict__ keys,
                                           unsigned long long* __restrict__ offers, const int* s_idx,
                                           const uint32_t* s_thr, int a, int b, uint32_t db) {
  const int ia = s_idx[a], ib = s_idx[b];
  const unsigned long long to_a = ((unsigned long long)db << 32) | (uint32_t)ib;
  const unsigned long long to_b = ((unsigned long long)db << 32) | (uint32_t)ia;
  if (db < s_thr[a] && !in_list<KB>(keys + (int64_t)ia * KB, to_a)) reservoir_insert(offers + (int64_t)ia * kRes, kRes, to_a);
  if (db < s_thr[b] && !in_list<KB>(keys + (int64_t)ib * KB, to_b)) reservoir_insert(offers + (int64_t)ib * kRes, kRes, to_b);
}

// ---------------------------------------------------------------------------------------------------------------
// join of dense rows: one CTA per row u.  The candidates (join_candidates) are staged in shared memory 64 features at
// a time; thread t < 100 owns the 4 x 4 pair tile (ta, tb), ta < 8 <= ... tb: every pair with a new member and a < b.
// ---------------------------------------------------------------------------------------------------------------
template <int KB, class T>
__global__ void __launch_bounds__(kJoinThreads)
nnd_join_kernel(const T* __restrict__ X, int64_t n, int d, const unsigned long long* __restrict__ keys,
                const int32_t* __restrict__ fwd, unsigned long long* __restrict__ rev, const uint32_t* __restrict__ thr,
                unsigned long long* __restrict__ offers) {
  __shared__ int s_raw[kCand];
  __shared__ int s_idx[kCand];
  __shared__ uint32_t s_thr[kCand];
  __shared__ int s_cnt[2];
  __shared__ float s_x[kCand][kFC + 1];  // odd row stride: the tiles' column reads hit distinct banks
  const int t = threadIdx.x;
  const int64_t u = blockIdx.x;
  join_candidates(u, fwd, rev, thr, s_raw, s_idx, s_thr, s_cnt);
  const int nn = s_cnt[0], no = s_cnt[1];
  if (nn == 0) return;  // nothing new around u
  auto slot_valid = [&](int r) { return r < 32 ? r < nn : r - 32 < no; };
  int ta = 0, tb = 0;
  {
    int q = t;
    while (ta < 8 && q >= 16 - ta) { q -= 16 - ta; ++ta; }
    tb = ta + q;
  }
  const bool active = t < kJoinTiles && 4 * ta < nn && slot_valid(4 * tb);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
  for (int f0 = 0; f0 < d; f0 += kFC) {
    const int fc = min(kFC, d - f0);
    __syncthreads();  // the previous chunk is consumed
    for (int e = t; e < kCand * kFC; e += kJoinThreads) {
      const int r = e / kFC, f = e % kFC;
      s_x[r][f] = (f < fc && slot_valid(r)) ? load_f32(X + (int64_t)s_idx[r] * d + f0 + f) : 0.0f;
    }
    __syncthreads();
    if (active) {
#pragma unroll 4
      for (int f = 0; f < fc; ++f) {
        float xa[4], xb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { xa[i] = s_x[4 * ta + i][f]; xb[i] = s_x[4 * tb + i][f]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) { const float df = xa[i] - xb[j]; acc[i][j] = fmaf(df, df, acc[i][j]); }
      }
    }
  }
  if (!active) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int a = 4 * ta + i, b = 4 * tb + j;
      if ((ta == tb && j <= i) || a >= nn || !slot_valid(b)) continue;
      offer_pair<KB>(keys, offers, s_idx, s_thr, a, b, __float_as_uint(acc[i][j]));
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// join of CSR rows: one CTA per row u, the candidates of join_candidates.  Their (column, value) slices are staged in
// shared memory in slot order (new rows first) while they fit kCsrStage entries; a row that does not fit is merged
// from global memory (same values, same sum).  One thread per pair: the nn (nn - 1) / 2 new-new pairs, then the
// nn x no new-old pairs, each one sequential merge.
// ---------------------------------------------------------------------------------------------------------------
template <int KB>
__global__ void __launch_bounds__(kCsrJoinThreads)
nnd_csr_join_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ cols,
                    const float* __restrict__ vals, const unsigned long long* __restrict__ keys,
                    const int32_t* __restrict__ fwd, unsigned long long* __restrict__ rev,
                    const uint32_t* __restrict__ thr, unsigned long long* __restrict__ offers) {
  __shared__ int s_raw[kCand];
  __shared__ int s_idx[kCand];
  __shared__ uint32_t s_thr[kCand];
  __shared__ int s_cnt[2];
  __shared__ int64_t s_beg[kCand];  // the slot's row in cols / vals
  __shared__ int s_len[kCand];
  __shared__ int s_off[kCand];      // its offset in s_col / s_val, or -1: read from global memory
  __shared__ int32_t s_col[kCsrStage];
  __shared__ float s_val[kCsrStage];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t u = blockIdx.x;
  join_candidates(u, fwd, rev, thr, s_raw, s_idx, s_thr, s_cnt);
  const int nn = s_cnt[0], no = s_cnt[1];
  if (nn == 0) return;  // nothing new around u
  if (t < kCand) {
    int64_t b = 0;
    int len = 0;
    if (t < 32 ? t < nn : t - 32 < no) { b = indptr[s_idx[t]]; len = (int)(indptr[s_idx[t] + 1] - b); }
    s_beg[t] = b;
    s_len[t] = len;
  }
  __syncthreads();
  if (t == 0) {
    int used = 0;
    for (int r = 0; r < kCand; ++r) {
      const int len = s_len[r];
      s_off[r] = len <= kCsrStage - used ? used : -1;
      if (s_off[r] >= 0) used += len;
    }
  }
  __syncthreads();
  for (int r = warp; r < kCand; r += kCsrJoinThreads / 32) {
    const int off = s_off[r], len = s_len[r];
    if (off < 0) continue;
    const int64_t b = s_beg[r];
    for (int e = lane; e < len; e += 32) { s_col[off + e] = __ldg(cols + b + e); s_val[off + e] = __ldg(vals + b + e); }
  }
  __syncthreads();
  const int p1 = nn * (nn - 1) / 2, total = p1 + nn * no;
  for (int p = t; p < total; p += kCsrJoinThreads) {
    int a, b;
    if (p < p1) {  // p = b (b - 1) / 2 + a, 0 <= a < b < nn
      b = (int)((1.0f + sqrtf(1.0f + 8.0f * (float)p)) * 0.5f);
      while (b * (b - 1) / 2 > p) --b;
      while ((b + 1) * b / 2 <= p) ++b;
      a = p - b * (b - 1) / 2;
    } else {
      const int q = p - p1;
      a = q / no;
      b = 32 + q % no;
    }
    const int oa = s_off[a], ob = s_off[b];
    const int32_t* ca = oa >= 0 ? s_col + oa : cols + s_beg[a];
    const float* va = oa >= 0 ? s_val + oa : vals + s_beg[a];
    const int32_t* cb = ob >= 0 ? s_col + ob : cols + s_beg[b];
    const float* vb = ob >= 0 ? s_val + ob : vals + s_beg[b];
    const float dist = (float)merge_dist2_rows(ca, va, s_len[a], cb, vb, s_len[b]);
    offer_pair<KB>(keys, offers, s_idx, s_thr, a, b, __float_as_uint(dist));
  }
}

// ---------------------------------------------------------------------------------------------------------------
// merge: one warp per row.  New list = the KB smallest of (list, offers not in the list, each once); entries from
// offers are flagged new and counted in *changes.  Resets the row's offer reservoir and writes the threshold of the
// next join (distance bits of the worst entry).
// ---------------------------------------------------------------------------------------------------------------
template <int KB>
__global__ void __launch_bounds__(256)
nnd_merge_kernel(int64_t n, unsigned long long* __restrict__ keys, uint8_t* __restrict__ flags,
                 uint32_t* __restrict__ thr, unsigned long long* __restrict__ offers,
                 unsigned long long* __restrict__ changes) {
  __shared__ unsigned long long s_l[8][KB];
  __shared__ unsigned long long s_r[8][kRes];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int64_t row = (int64_t)blockIdx.x * 8 + w;
  if (row >= n) return;
  constexpr int P = KB / 32;
  uint8_t fl[P];
#pragma unroll
  for (int s = 0; s < P; ++s) {
    const int j = lane + 32 * s;
    s_l[w][j] = keys[row * KB + j];
    fl[s] = flags[row * KB + j];
  }
  const unsigned long long x = offers[row * kRes + lane];
  offers[row * kRes + lane] = kEmpty;
  s_r[w][lane] = x;
  __syncwarp();
  // lower bound of x in the list
  int lo = 0, hi = KB;
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (s_l[w][mid] < x) lo = mid + 1; else hi = mid; }
  const bool fresh = x != kEmpty && (lane == 0 || s_r[w][lane - 1] != x) && !(lo < KB && s_l[w][lo] == x);
  const unsigned vmask = __ballot_sync(kFull, fresh);
  const int pos_x = lo + __popc(vmask & ((1u << lane) - 1));
  const bool enters = fresh && pos_x < KB;
  if (enters) {
    keys[row * KB + pos_x] = x;
    flags[row * KB + pos_x] = 1;
    if (pos_x == KB - 1) thr[row] = (uint32_t)(x >> 32);
  }
#pragma unroll
  for (int s = 0; s < P; ++s) {
    const int j = lane + 32 * s;
    const unsigned long long key = s_l[w][j];
    int before = 0;
    for (int q = 0; q < kRes; ++q) before += ((vmask >> q) & 1u) && s_r[w][q] < key;
    const int pos = j + before;
    if (pos < KB) {
      keys[row * KB + pos] = key;
      flags[row * KB + pos] = fl[s];
      if (pos == KB - 1) thr[row] = (uint32_t)(key >> 32);
    }
  }
  const int changed = __popc(__ballot_sync(kFull, enters));
  if (lane == 0 && changed) atomicAdd(changes, (unsigned long long)changed);
}

// list keys -> the candidate indices read by the re-rank kernels (-1 for an empty slot)
__global__ void __launch_bounds__(256)
nnd_extract_kernel(int64_t count, const unsigned long long* __restrict__ keys, int32_t* __restrict__ cand) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const unsigned long long key = keys[i];
  cand[i] = key == kEmpty ? -1 : (int32_t)(uint32_t)key;
}

struct ApproxLayout {
  int kb;
  size_t off_keys, off_flags, off_thr, off_offers, off_rev, off_fwd, off_cand, off_changes, total;
};

ApproxLayout approx_layout(int64_t n, int k) {
  ApproxLayout L;
  L.kb = k <= kNarrowMaxK ? kNarrowKK : kWideKK;
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  const size_t nn = (size_t)n;
  size_t o = 0;
  L.off_keys = o; o = up(o + nn * L.kb * 8);
  L.off_flags = o; o = up(o + nn * L.kb);
  L.off_thr = o; o = up(o + nn * 4);
  L.off_offers = o; o = up(o + nn * kRes * 8);
  L.off_rev = o; o = up(o + nn * 2 * kS * 8);
  L.off_fwd = o; o = up(o + nn * 2 * kS * 4);
  L.off_cand = o; o = up(o + nn * L.kb * 4);
  L.off_changes = o; o = up(o + 8);
  L.total = o;
  return L;
}

// CSR search: prepare_csr's workspace (without candidate lists), then the lists.  The workspace size is host
// arithmetic alone, so the sort scratch is reserved as csr_sort_scratch_bound; the call checks CUB's exact figure
// against it.
struct ApproxCsrLayout {
  CsrKnnLayout prep;
  ApproxLayout lists;  // offsets from prep.total
  size_t total;
};

ApproxCsrLayout approx_csr_layout(int64_t n, int d, int64_t nnz, int k) {
  ApproxCsrLayout A;
  csr_knn_carve(n, d, nnz, 0, csr_sort_scratch_bound(d, nnz), &A.prep);
  A.lists = approx_layout(n, k);
  A.total = A.prep.total + A.lists.total;
  return A;
}

// The format-specific launches of the driver.
template <int KB, class T>
int launch_join(const DenseRows<T>& r, int64_t n, const unsigned long long* keys, const int32_t* fwd,
                unsigned long long* rev, const uint32_t* thr, unsigned long long* offers, cudaStream_t st) {
  nnd_join_kernel<KB, T><<<(unsigned)n, kJoinThreads, 0, st>>>(r.X, n, r.d, keys, fwd, rev, thr, offers);
  MDE_LAUNCH_CHECK();
  return 0;
}
template <int KB>
int launch_join(const CsrRows& r, int64_t n, const unsigned long long* keys, const int32_t* fwd,
                unsigned long long* rev, const uint32_t* thr, unsigned long long* offers, cudaStream_t st) {
  nnd_csr_join_kernel<KB><<<(unsigned)n, kCsrJoinThreads, 0, st>>>(r.indptr, r.cols, r.vals, keys, fwd, rev, thr,
                                                                    offers);
  MDE_LAUNCH_CHECK();
  return 0;
}
template <int KB, class T>
int launch_rerank(const DenseRows<T>& r, int64_t n, const int32_t* cand, int k, int32_t* idx_out, float* d2_out,
                  cudaStream_t st) {
  return knn_dense_rerank<T>(KB, r.X, n, r.d, cand, k, idx_out, d2_out, st);
}
template <int KB>
int launch_rerank(const CsrRows& r, int64_t n, const int32_t* cand, int k, int32_t* idx_out, float* d2_out,
                  cudaStream_t st) {
  const unsigned grid = (unsigned)((n + 7) / 8);
  if (KB == kNarrowKK)
    knn_csr_rerank_kernel<<<grid, 256, 0, st>>>(r.indptr, r.cols, r.vals, 0, n, cand, k, idx_out, d2_out);
  else knn_csr_wide_rerank_kernel<<<grid, 256, 0, st>>>(r.indptr, r.cols, r.vals, 0, n, cand, k, idx_out, d2_out);
  MDE_LAUNCH_CHECK();
  return 0;
}

template <int KB, class Rows>
int run_approx(const Rows& rows, int64_t n, int k, uint64_t seed, int32_t* idx_out, float* d2_out, uint8_t* w,
               const ApproxLayout& L, cudaStream_t st, int* iterations) {
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(w + L.off_keys);
  uint8_t* flags = w + L.off_flags;
  uint32_t* thr = reinterpret_cast<uint32_t*>(w + L.off_thr);
  unsigned long long* offers = reinterpret_cast<unsigned long long*>(w + L.off_offers);
  unsigned long long* rev = reinterpret_cast<unsigned long long*>(w + L.off_rev);
  int32_t* fwd = reinterpret_cast<int32_t*>(w + L.off_fwd);
  int32_t* cand = reinterpret_cast<int32_t*>(w + L.off_cand);
  unsigned long long* changes = reinterpret_cast<unsigned long long*>(w + L.off_changes);
  const unsigned warp_grid = (unsigned)((n + 7) / 8);
  nnd_init_kernel<KB, Rows><<<warp_grid, 256, 0, st>>>(rows, n, seed, keys, flags, thr, offers, rev);
  MDE_LAUNCH_CHECK();
  int max_iter = 5;
  while ((1ll << max_iter) < n) ++max_iter;  // max(5, ceil(log2 n))
  int it = 0;
  if (n - 1 > KB) {  // else every list already holds every other row
    for (; it < max_iter;) {
      MDE_CUDA_TRY(cudaMemsetAsync(changes, 0, sizeof(unsigned long long), st));
      nnd_sample_kernel<KB><<<warp_grid, 256, 0, st>>>(n, seed, it, keys, flags, fwd, rev);
      MDE_LAUNCH_CHECK();
      int rc;
      if ((rc = launch_join<KB>(rows, n, keys, fwd, rev, thr, offers, st))) return rc;
      nnd_merge_kernel<KB><<<warp_grid, 256, 0, st>>>(n, keys, flags, thr, offers, changes);
      MDE_LAUNCH_CHECK();
      unsigned long long changed = 0;
      MDE_CUDA_TRY(cudaMemcpyAsync(&changed, changes, sizeof(changed), cudaMemcpyDeviceToHost, st));
      MDE_CUDA_TRY(cudaStreamSynchronize(st));
      ++it;
      if (changed * kDeltaInv < (unsigned long long)n * KB) break;
    }
  }
  if (iterations) *iterations = it;
  const int64_t count = n * KB;
  nnd_extract_kernel<<<(unsigned)((count + 255) / 256), 256, 0, st>>>(count, keys, cand);
  MDE_LAUNCH_CHECK();
  return launch_rerank<KB>(rows, n, cand, k, idx_out, d2_out, st);
}

// The dense search on a matrix of element type T.
template <class T>
int approx_dense(const T* X, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws,
                 size_t ws_bytes, void* stream, int* iterations) {
  if (!X || !idx_out || !d2_out || !ws || n < 2 || d < 1 || k < 1 || k > kWideMaxK || k > n - 1)
    return MDE_E_INVALID;
  if (n >= (1ll << 31) - 128) return MDE_E_UNSUPPORTED;
  const ApproxLayout L = approx_layout(n, k);
  if (ws_bytes < L.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = static_cast<uint8_t*>(ws);
  const DenseRows<T> rows{X, d};
  if (L.kb == kNarrowKK) return run_approx<kNarrowKK>(rows, n, k, seed, idx_out, d2_out, w, L, st, iterations);
  return run_approx<kWideKK>(rows, n, k, seed, idx_out, d2_out, w, L, st, iterations);
}

}  // namespace

extern "C" {

int mde_knn_approx_max_k(void) { return kWideMaxK; }

int mde_knn_approx_ws_bytes(int64_t n, int d, int k, size_t* bytes) {
  if (!bytes || n < 2 || d < 1 || k < 1 || k > kWideMaxK || k > n - 1) return MDE_E_INVALID;
  *bytes = approx_layout(n, k).total;
  return 0;
}

int mde_knn_approx_ex(const float* X, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out, float* d2_out,
                      void* ws, size_t ws_bytes, void* stream, int* iterations) {
  return approx_dense<float>(X, n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream, iterations);
}

int mde_knn_approx(const float* X, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws,
                   size_t ws_bytes, void* stream) {
  return mde_knn_approx_ex(X, n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn16_approx_ws_bytes(int64_t n, int d, int k, size_t* bytes) { return mde_knn_approx_ws_bytes(n, d, k, bytes); }

int mde_knn16_approx_ex(const void* X, int dtype, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out,
                        float* d2_out, void* ws, size_t ws_bytes, void* stream, int* iterations) {
  if (dtype == MDE_DTYPE_FP16)
    return approx_dense<__half>(static_cast<const __half*>(X), n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream,
                                iterations);
  if (dtype == MDE_DTYPE_BF16)
    return approx_dense<__nv_bfloat16>(static_cast<const __nv_bfloat16*>(X), n, d, k, seed, idx_out, d2_out, ws,
                                       ws_bytes, stream, iterations);
  return MDE_E_INVALID;
}

int mde_knn16_approx(const void* X, int dtype, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out,
                     float* d2_out, void* ws, size_t ws_bytes, void* stream) {
  return mde_knn16_approx_ex(X, dtype, n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn8_approx_ws_bytes(int64_t n, int d, int k, size_t* bytes) { return mde_knn_approx_ws_bytes(n, d, k, bytes); }

int mde_knn8_approx_ex(const void* X, int dtype, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out,
                       float* d2_out, void* ws, size_t ws_bytes, void* stream, int* iterations) {
  if (dtype == MDE_DTYPE_U8)
    return approx_dense<uint8_t>(static_cast<const uint8_t*>(X), n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream,
                                 iterations);
  if (dtype == MDE_DTYPE_S8)
    return approx_dense<int8_t>(static_cast<const int8_t*>(X), n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream,
                                iterations);
  return MDE_E_INVALID;
}

int mde_knn8_approx(const void* X, int dtype, int64_t n, int d, int k, uint64_t seed, int32_t* idx_out,
                    float* d2_out, void* ws, size_t ws_bytes, void* stream) {
  return mde_knn8_approx_ex(X, dtype, n, d, k, seed, idx_out, d2_out, ws, ws_bytes, stream, nullptr);
}

int mde_knn_approx_csr_ws_bytes(int64_t n, int d, int64_t nnz, int k, size_t* bytes) {
  if (!bytes || n < 2 || d < 1 || nnz < 0 || k < 1 || k > kWideMaxK || k > n - 1) return MDE_E_INVALID;
  *bytes = approx_csr_layout(n, d, nnz, k).total;
  return 0;
}

int mde_knn_approx_csr_ex(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                          int64_t nnz, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws,
                          size_t ws_bytes, void* stream, int* iterations) {
  if (!indptr || !idx_out || !d2_out || !ws || n < 2 || d < 1 || nnz < 0 || k < 1 || k > kWideMaxK || k > n - 1)
    return MDE_E_INVALID;
  if (nnz > 0 && (!indices || !values)) return MDE_E_INVALID;
  if (n >= (1ll << 31) - 128) return MDE_E_UNSUPPORTED;
  const ApproxCsrLayout A = approx_csr_layout(n, d, nnz, k);
  if (ws_bytes < A.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  size_t sort_bytes = 0;
  int rc = csr_sort_scratch(n, d, nnz, &sort_bytes);
  if (rc) return rc;
  if (sort_bytes > A.prep.tmp_bytes) return MDE_E_ALLOC;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = static_cast<uint8_t*>(ws);
  if ((rc = prepare_csr(indptr, indices, values, n, d, nnz, A.prep, w, st))) return rc;
  const CsrRows rows{indptr, reinterpret_cast<const int32_t*>(w + A.prep.off_kin),
                     reinterpret_cast<const float*>(w + A.prep.off_val)};
  uint8_t* wl = w + A.prep.total;
  if (A.lists.kb == kNarrowKK)
    return run_approx<kNarrowKK>(rows, n, k, seed, idx_out, d2_out, wl, A.lists, st, iterations);
  return run_approx<kWideKK>(rows, n, k, seed, idx_out, d2_out, wl, A.lists, st, iterations);
}

int mde_knn_approx_csr(const int64_t* indptr, const int32_t* indices, const float* values, int64_t n, int d,
                       int64_t nnz, int k, uint64_t seed, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
                       void* stream) {
  return mde_knn_approx_csr_ex(indptr, indices, values, n, d, nnz, k, seed, idx_out, d2_out, ws, ws_bytes, stream,
                               nullptr);
}

}  // extern "C"
