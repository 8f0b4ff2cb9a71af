// mde_graph.cu -- hop-count shortest paths of an unweighted graph on the device (SURVEY section 8 row f4).
//
// Replaces pymde/preprocess/graph.py:310-474 for unweighted graphs: the reference runs ONE breadth-first search
// per node (Cython, pymde/preprocess/_graph.pyx:10-52) in a multiprocessing pool and keeps, for node s, the
// distances to the nodes v > s, each with probability `retain_fraction`.
//
// Here the searches are bit-parallel: a batch of 256 sources advances together, node v holding 4 x 64-bit words of
// "reached by source b" bits.  One level is one pass over the CSR adjacency:
//     next[v] = (OR over neighbours u of frontier[u]) & ~visited[v]
// (64 sources per 8-byte load, no atomics on the frontier), and every newly set bit (s, v) with v > s is a
// finished shortest path of `level` hops; it is kept when a counter-based hash of (seed, s, v) falls under
// `retain` and appended through one warp-aggregated atomic per warp.  The output order depends on the schedule
// (the SET of triples does not); the caller sorts by (s, v).
//
// Weighted graphs (mde_graph_sssp) and the graph k-nearest neighbours (mde_graph_knn) use a frontier-driven
// Bellman-Ford engine further down.
#include <cstdint>
#include <cstdlib>

#include <cooperative_groups.h>

#include "mde_common.cuh"

using namespace mde;
namespace cg = cooperative_groups;

namespace {

constexpr int kWords = 4;               // 64-bit words per node: 256 sources per batch
constexpr int kBatch = 64 * kWords;

__device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}

__global__ void hops_init_kernel(uint64_t* __restrict__ visited, uint64_t* __restrict__ front, int64_t n,
                                 int64_t s0, int nsrc) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n * kWords) return;
  const int64_t v = k / kWords;
  const int w = (int)(k % kWords);
  uint64_t bits = 0ull;
  const int64_t b = v - s0;  // source b of the batch is node s0 + b
  if (b >= 0 && b < nsrc && (b >> 6) == w) bits = 1ull << (b & 63);
  visited[k] = bits;
  front[k] = bits;
}

__global__ void __launch_bounds__(256)
hops_level_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                  const uint64_t* __restrict__ front_in, uint64_t* __restrict__ visited,
                  uint64_t* __restrict__ front_out, int64_t n, int64_t s0, int level, int emit, uint64_t seed,
                  uint64_t thresh, int32_t* __restrict__ out_src, int32_t* __restrict__ out_dst,
                  float* __restrict__ out_len, int64_t cap, unsigned long long* __restrict__ count,
                  int* __restrict__ any) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = threadIdx.x & 31;
  uint64_t fresh = 0ull;
  int64_t v = 0;
  int w = 0;
  if (k < n * kWords) {
    v = k / kWords;
    w = (int)(k % kWords);
    uint64_t acc = 0ull;
    const int e0 = indptr[v], e1 = indptr[v + 1];
    for (int e = e0; e < e1; ++e) acc |= front_in[(int64_t)indices[e] * kWords + w];
    fresh = acc & ~visited[k];
    front_out[k] = fresh;
    if (fresh) { visited[k] |= fresh; *any = 1; }
  }
  if (!emit) return;
  // finished paths (s, v), v > s, kept with probability thresh / 2^64
  uint64_t keep = 0ull;
  uint64_t bits = fresh;
  while (bits) {
    const int b = __ffsll((long long)bits) - 1;
    bits &= bits - 1;
    const int64_t s = s0 + 64 * w + b;
    if (v > s && (thresh == ~0ull || splitmix64(seed ^ ((uint64_t)s * (uint64_t)n + (uint64_t)v)) < thresh))
      keep |= 1ull << b;
  }
  const int cnt = __popcll(keep);
  // warp-aggregated append
  int incl = cnt;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int o = __shfl_up_sync(kFull, incl, off);
    if (lane >= off) incl += o;
  }
  const int total = __shfl_sync(kFull, incl, 31);
  unsigned long long base = 0ull;
  if (lane == 31 && total > 0) base = atomicAdd(count, (unsigned long long)total);
  base = __shfl_sync(kFull, base, 31);
  unsigned long long pos = base + (unsigned long long)(incl - cnt);
  while (keep) {
    const int b = __ffsll((long long)keep) - 1;
    keep &= keep - 1;
    if ((int64_t)pos < cap) {
      out_src[pos] = (int32_t)(s0 + 64 * w + b);
      out_dst[pos] = (int32_t)v;
      out_len[pos] = (float)level;
    }
    ++pos;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// Weighted shortest paths (mde_graph_sssp) and graph k-nearest neighbours (mde_graph_knn).
//
// Algorithm: frontier-driven Bellman-Ford over a batch of B sources.  The batch owns one distance tile
// dist[v * B + b] (fp64 bit patterns; ~0 = not reached).  A queue holds the (node, source) entries improved in the
// last round; one thread per entry pushes its length to the node's neighbours with a 64-bit atomicMin.  Non-negative
// doubles order like their unsigned bit patterns, x -> fl(x + w) is monotone and never decreases for w >= 0, so any
// relaxation order reaches the same least fixed point: per node, the minimum fp64 fold-sum over paths -- exactly what
// scipy's Dijkstra computes on the float64-widened weights.  The result is schedule-free, bit for bit.  Chosen over
// delta-stepping for its simplicity: the recipes' searches are either radius-bounded (k-NN: a few rounds) or
// sampled all-pairs, where every (source, node) entry is settled anyway and the extra re-relaxations of plain
// Bellman-Ford stay a small factor.
//
// Locality: nothing per batch costs O(n * B) unless the search touches that many entries.  Every entry reached for
// the first time (atomicMin returns ~0) is appended once to a `touched` list; emission, k-NN selection and the reset
// of the tile for the next batch walk that list.  The tile and the queue stamps are initialised once per call.
// A per-entry stamp (the round that last queued it) keeps each entry at most once in a queue, so every queue fits in
// n * B slots.  Queue entries are packed (v << 32) | b.
// ------------------------------------------------------------------------------------------------------------------
constexpr unsigned long long kUnreached = ~0ull;
constexpr int kRelaxThreads = 256;
constexpr int kRelaxBlocks = kNumSMs * 8;   // fixed grid: the queue length lives on the device
constexpr int kRoundsPerCheck = 4;          // rounds launched between two reads of the queue length
constexpr int kKnnMaxK = 64;

// device-side counters: queue lengths (3-slot rotation, see sssp_relax_kernel) and the touched-list length
struct PathCounters {
  unsigned long long queue[3];
  unsigned long long touched;
};

struct PathWs {
  PathCounters* ctr;
  unsigned long long* dist;   // [n * B]
  uint64_t* touched;          // [n * B] packed entries
  uint64_t* queue[2];         // [n * B] each; after convergence queue[0] doubles as the k-NN segment buffer
  int* stamp;                 // [n * B]
  int* seg_count;             // [B]
  unsigned long long* seg_off;  // [B + 1]
  unsigned long long* seg_cur;  // [B]
};

constexpr int64_t kMaxBatch = 1 << 20;

inline int64_t align_up(int64_t x) { return (x + 255) & ~int64_t(255); }

inline int64_t path_ws_bytes(int64_t n, int64_t B) {
  const int64_t nb = n * B;
  return align_up(sizeof(PathCounters)) + 4 * align_up(nb * 8) + align_up(nb * 4) + align_up(B * 4) +
         align_up(B * 8) + align_up((B + 1) * 8) + 256;
}

// largest multiple of 32 (at most the rounded-up source count) whose workspace fits; 0 if not even 32 fits
inline int64_t path_batch(int64_t n, int64_t nsrc, int64_t ws_bytes) {
  int64_t most = ((nsrc + 31) / 32) * 32;
  if (most > kMaxBatch) most = kMaxBatch;
  if (ws_bytes < path_ws_bytes(n, 32)) return 0;
  int64_t lo = 32, hi = most < 32 ? 32 : most;
  while (lo < hi) {  // binary search over multiples of 32
    const int64_t mid = ((lo + hi + 32) / 64) * 32;
    if (mid > lo && path_ws_bytes(n, mid) <= ws_bytes) lo = mid; else hi = mid - 32;
  }
  return lo;
}

inline PathWs path_ws(void* ws, int64_t n, int64_t B) {
  uintptr_t p = ((uintptr_t)ws + 255) & ~uintptr_t(255);
  const int64_t nb = n * B;
  PathWs w;
  w.ctr = reinterpret_cast<PathCounters*>(p); p += align_up(sizeof(PathCounters));
  w.dist = reinterpret_cast<unsigned long long*>(p); p += align_up(nb * 8);
  w.touched = reinterpret_cast<uint64_t*>(p); p += align_up(nb * 8);
  w.queue[0] = reinterpret_cast<uint64_t*>(p); p += align_up(nb * 8);
  w.queue[1] = reinterpret_cast<uint64_t*>(p); p += align_up(nb * 8);
  w.stamp = reinterpret_cast<int*>(p); p += align_up(nb * 4);
  w.seg_count = reinterpret_cast<int*>(p); p += align_up(B * 4);
  w.seg_cur = reinterpret_cast<unsigned long long*>(p); p += align_up(B * 8);
  w.seg_off = reinterpret_cast<unsigned long long*>(p);
  return w;
}

// warp-aggregated append: one atomic per group of lanes that reach the call together
__device__ __forceinline__ unsigned long long append_slot(unsigned long long* ctr) {
  cg::coalesced_group g = cg::coalesced_threads();
  unsigned long long base = 0ull;
  if (g.thread_rank() == 0) base = atomicAdd(ctr, (unsigned long long)g.size());
  return g.shfl(base, 0) + g.thread_rank();
}

__global__ void sssp_seed_kernel(PathWs w, int64_t B, int64_t s0, int nsrc) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b == 0) {
    w.ctr->queue[1] = (unsigned long long)nsrc;  // round 1 reads slot 1 and appends to slot 2
    w.ctr->queue[2] = 0ull;
    w.ctr->touched = (unsigned long long)nsrc;
  }
  if (b >= nsrc) return;
  const int64_t v = s0 + b;
  const uint64_t e = ((uint64_t)v << 32) | (uint32_t)b;
  w.dist[v * B + b] = 0ull;  // bit pattern of +0.0
  w.stamp[v * B + b] = 1;
  w.touched[b] = e;
  w.queue[1][b] = e;
}

// Round r: relax every entry queued for round r (queue[r & 1], length in slot r % 3) and queue the improved entries
// for round r + 1 (queue[(r + 1) & 1], slot (r + 1) % 3).  Slot (r + 2) % 3 was round r - 1's input and is zeroed
// here for round r + 1's appends, so rounds run back to back without host work in between.
__global__ void __launch_bounds__(kRelaxThreads)
sssp_relax_kernel(const int32_t* __restrict__ indptr, const int32_t* __restrict__ indices,
                  const float* __restrict__ weights, PathWs w, int64_t B, double max_len, int round) {
  const unsigned long long nin = w.ctr->queue[round % 3];
  unsigned long long* nout = &w.ctr->queue[(round + 1) % 3];
  if (blockIdx.x == 0 && threadIdx.x == 0) w.ctr->queue[(round + 2) % 3] = 0ull;
  // (a select, not w.queue[round & 1]: indexing the by-value parameter array would copy it to the stack)
  const uint64_t* __restrict__ qin = (round & 1) ? w.queue[1] : w.queue[0];
  uint64_t* __restrict__ qout = (round & 1) ? w.queue[0] : w.queue[1];
  const int next = round + 1;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nin;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t e = qin[i];
    const int64_t u = (int64_t)(e >> 32);
    const int64_t b = (int64_t)(e & 0xffffffffull);
    const double du = __longlong_as_double((long long)w.dist[u * B + b]);
    const int p0 = indptr[u], p1 = indptr[u + 1];
    for (int p = p0; p < p1; ++p) {
      const int64_t v = indices[p];
      const double nd = du + (weights ? (double)weights[p] : 1.0);
      if (!(nd <= max_len)) continue;
      const unsigned long long bits = (unsigned long long)__double_as_longlong(nd);
      unsigned long long* slot = &w.dist[v * B + b];
      if (bits >= *slot) continue;  // a stale read is never below the current value: safe to skip
      const unsigned long long old = atomicMin(slot, bits);
      if (bits >= old) continue;
      const uint64_t ev = ((uint64_t)v << 32) | (uint64_t)b;
      if (old == kUnreached) w.touched[append_slot(&w.ctr->touched)] = ev;
      if (atomicExch(&w.stamp[v * B + b], next) != next) qout[append_slot(nout)] = ev;
    }
  }
}

// Shortest-path emission (same rule and hash as hops_level_kernel) fused with the reset of the touched entries.
__global__ void __launch_bounds__(256)
sssp_emit_reset_kernel(PathWs w, int64_t B, int64_t n, int64_t s0, uint64_t seed, uint64_t thresh,
                       int32_t* __restrict__ out_src, int32_t* __restrict__ out_dst, float* __restrict__ out_len,
                       int64_t cap, unsigned long long* __restrict__ count) {
  const unsigned long long nt = w.ctr->touched;
  const int lane = threadIdx.x & 31;
  const unsigned long long warp0 = ((unsigned long long)blockIdx.x * blockDim.x + threadIdx.x) & ~31ull;
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  for (unsigned long long base = warp0; base < nt; base += stride) {  // warp-uniform trip count
    const unsigned long long i = base + lane;
    bool keep = false;
    int64_t s = 0, v = 0;
    float len = 0.0f;
    if (i < nt) {
      const uint64_t e = w.touched[i];
      v = (int64_t)(e >> 32);
      const int64_t b = (int64_t)(e & 0xffffffffull);
      s = s0 + b;
      len = (float)__longlong_as_double((long long)w.dist[v * B + b]);
      w.dist[v * B + b] = kUnreached;
      w.stamp[v * B + b] = 0;
      keep = v > s && (thresh == ~0ull || splitmix64(seed ^ ((uint64_t)s * (uint64_t)n + (uint64_t)v)) < thresh);
    }
    const unsigned ballot = __ballot_sync(kFull, keep);
    unsigned long long pos = 0ull;
    if (lane == 0 && ballot) pos = atomicAdd(count, (unsigned long long)__popc(ballot));
    pos = __shfl_sync(kFull, pos, 0) + (unsigned long long)__popc(ballot & ((1u << lane) - 1u));
    if (keep && (int64_t)pos < cap) {
      out_src[pos] = (int32_t)s;
      out_dst[pos] = (int32_t)v;
      out_len[pos] = len;
    }
  }
}

// k-NN selection, step 1: entries per source (the source itself excluded)
__global__ void knn_count_kernel(PathWs w, int64_t s0) {
  const unsigned long long nt = w.ctr->touched;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nt;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t e = w.touched[i];
    const int64_t b = (int64_t)(e & 0xffffffffull);
    if ((int64_t)(e >> 32) != s0 + b) atomicAdd(&w.seg_count[b], 1);
  }
}

// step 2: exclusive scan of the B counts (one block of 1024 threads, contiguous chunks per thread)
__global__ void __launch_bounds__(1024) knn_scan_kernel(PathWs w, int B) {
  __shared__ unsigned long long warp_tot[32];
  const int t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int chunk = (B + 1023) / 1024;
  const int c0 = t * chunk, c1 = min(B, c0 + chunk);
  unsigned long long sum = 0ull;
  for (int c = c0; c < c1; ++c) sum += (unsigned long long)w.seg_count[c];
  unsigned long long incl = sum;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const unsigned long long o = __shfl_up_sync(kFull, incl, off);
    if (lane >= off) incl += o;
  }
  if (lane == 31) warp_tot[wid] = incl;
  __syncthreads();
  if (wid == 0) {
    unsigned long long x = warp_tot[lane];
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const unsigned long long o = __shfl_up_sync(kFull, x, off);
      if (lane >= off) x += o;
    }
    warp_tot[lane] = x;  // inclusive over warps
  }
  __syncthreads();
  unsigned long long run = incl - sum + (wid > 0 ? warp_tot[wid - 1] : 0ull);
  for (int c = c0; c < c1; ++c) {
    w.seg_off[c] = run;
    w.seg_cur[c] = run;
    run += w.seg_count[c];
  }
  if (t == 1023) w.seg_off[B] = warp_tot[31];
}

// step 3: node indices grouped by source (order within a group is irrelevant: selection keys are unique)
__global__ void knn_scatter_kernel(PathWs w, int64_t s0) {
  const unsigned long long nt = w.ctr->touched;
  int32_t* seg = reinterpret_cast<int32_t*>(w.queue[0]);
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nt;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t e = w.touched[i];
    const int64_t v = (int64_t)(e >> 32), b = (int64_t)(e & 0xffffffffull);
    if (v != s0 + b) seg[atomicAdd(&w.seg_cur[b], 1ull)] = (int32_t)v;
  }
}

__device__ __forceinline__ bool key_less(unsigned long long d0, int v0, unsigned long long d1, int v1) {
  return d0 < d1 || (d0 == d1 && v0 < v1);
}

// step 4: one warp per source; k rounds of a warp-wide minimum of (length, node) above the last one chosen.
// Source s0 + b is written to output row s0 + b - row0 (row0: the first source of the call's range).
__global__ void __launch_bounds__(256)
knn_select_kernel(PathWs w, int64_t B, int64_t s0, int64_t row0, int nsrc, int k, int32_t* __restrict__ out_idx,
                  float* __restrict__ out_len) {
  const int b = (int)(((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (b >= nsrc) return;
  const int32_t* seg = reinterpret_cast<const int32_t*>(w.queue[0]);
  const int64_t lo = (int64_t)w.seg_off[b], hi = (int64_t)w.seg_off[b + 1];
  unsigned long long last_d = 0ull;
  int last_v = -1;
  int32_t* oi = out_idx + (s0 - row0 + b) * (int64_t)k;
  float* ol = out_len + (s0 - row0 + b) * (int64_t)k;
  for (int j = 0; j < k; ++j) {
    unsigned long long best_d = kUnreached;
    int best_v = 0x7fffffff;
    for (int64_t i = lo + lane; i < hi; i += 32) {
      const int v = seg[i];
      const unsigned long long d = w.dist[(int64_t)v * B + b];
      if (key_less(last_d, last_v, d, v) && key_less(d, v, best_d, best_v)) { best_d = d; best_v = v; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned long long od = __shfl_xor_sync(kFull, best_d, off);
      const int ov = __shfl_xor_sync(kFull, best_v, off);
      if (key_less(od, ov, best_d, best_v)) { best_d = od; best_v = ov; }
    }
    if (lane == 0) {
      const bool found = best_d != kUnreached;
      oi[j] = found ? best_v : -1;
      ol[j] = found ? (float)__longlong_as_double((long long)best_d) : __int_as_float(0x7f800000);
    }
    last_d = best_d;
    last_v = best_v;
  }
}

// step 4 for 1 <= k <= kKnnLongMaxK (mde_graph_knn_long*): one CTA per source, the same lists as knn_select_kernel.
// A selection key is the 96-bit (fp64 length bits, node index) pair, unique within a source.  Segments of at most
// kLongSmem entries are sorted whole in shared memory.  Longer ones (a hub, an unlimited radius) never sit in shared
// memory: an MSB radix select, 8 bits per pass over the segment in global memory, finds the k-th key, starting below
// the common prefix of the segment's smallest and largest keys and stopping at the first digit whose bin holds exactly
// the keys still wanted; the <= k winners are then compacted into shared memory and sorted.  So the work per source is
// O(passes x segment) whatever k, and ties cost at most the 4 passes over the node-index bits.
constexpr int kKnnLongMaxK = 256;
constexpr int kLongThreads = 256;
constexpr int kLongSmem = 2048;   // keys sorted whole in shared memory: 24 KB

typedef unsigned __int128 u128;

__device__ __forceinline__ u128 long_key(const PathWs& w, int64_t B, int b, int v) {
  return ((u128)w.dist[(int64_t)v * B + b] << 32) | (uint32_t)v;
}

// ascending bitonic sort of sd / sv [0, len) in shared memory, len a power of two; ends with a barrier
__device__ void long_sort(unsigned long long* sd, int* sv, int len) {
  for (int size = 2; size <= len; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int i = threadIdx.x; i < (len >> 1); i += kLongThreads) {
        const int lo = 2 * stride * (i / stride) + (i % stride), hi = lo + stride;
        const bool up = (lo & size) == 0;
        if (key_less(sd[hi], sv[hi], sd[lo], sv[lo]) == up) {
          const unsigned long long td = sd[lo]; sd[lo] = sd[hi]; sd[hi] = td;
          const int tv = sv[lo]; sv[lo] = sv[hi]; sv[hi] = tv;
        }
      }
      __syncthreads();
    }
  }
}

__device__ __forceinline__ u128 shfl_xor_u128(u128 x, int off) {
  const unsigned long long hi = __shfl_xor_sync(kFull, (unsigned long long)(x >> 64), off);
  const unsigned long long lo = __shfl_xor_sync(kFull, (unsigned long long)x, off);
  return ((u128)hi << 64) | lo;
}

__global__ void __launch_bounds__(kLongThreads)
knn_select_long_kernel(PathWs w, int64_t B, int64_t s0, int64_t row0, int k, int32_t* __restrict__ out_idx,
                       float* __restrict__ out_len) {
  __shared__ unsigned long long sd[kLongSmem];
  __shared__ int sv[kLongSmem];
  __shared__ int hist[256];
  __shared__ u128 red[2][kLongThreads / 32];
  __shared__ int sel_bin, sel_below, sel_cnt, n_win;
  const int b = blockIdx.x, t = threadIdx.x, lane = t & 31, wid = t >> 5;
  const int32_t* seg = reinterpret_cast<const int32_t*>(w.queue[0]);
  const int64_t lo = (int64_t)w.seg_off[b], len = (int64_t)w.seg_off[b + 1] - lo;
  int m;  // keys in sd / sv to sort: the whole segment, or the k winners
  if (len <= kLongSmem) {
    for (int i = t; i < (int)len; i += kLongThreads) {
      const int v = seg[lo + i];
      sd[i] = w.dist[(int64_t)v * B + b];
      sv[i] = v;
    }
    m = (int)len;
  } else {
    // the smallest and largest key: every key shares their common prefix
    u128 kmin = ~(u128)0, kmax = 0;
    for (int64_t i = t; i < len; i += kLongThreads) {
      const u128 key = long_key(w, B, b, seg[lo + i]);
      kmin = key < kmin ? key : kmin;
      kmax = key > kmax ? key : kmax;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const u128 a = shfl_xor_u128(kmin, off), c = shfl_xor_u128(kmax, off);
      kmin = a < kmin ? a : kmin;
      kmax = c > kmax ? c : kmax;
    }
    if (lane == 0) { red[0][wid] = kmin; red[1][wid] = kmax; }
    __syncthreads();
    kmin = red[0][0]; kmax = red[1][0];
    for (int i = 1; i < kLongThreads / 32; ++i) {
      kmin = red[0][i] < kmin ? red[0][i] : kmin;
      kmax = red[1][i] > kmax ? red[1][i] : kmax;
    }
    // keys are distinct and len > k, so kmin != kmax; s is the digit holding the highest differing bit
    const u128 diff = kmin ^ kmax;
    const unsigned long long dh = (unsigned long long)(diff >> 64), dl = (unsigned long long)diff;
    const int top = dh ? 128 - __clzll((long long)dh) : 64 - __clzll((long long)dl);
    int s = ((top - 1) / 8) * 8;
    u128 prefix = (kmin >> (s + 8)) << (s + 8);
    int want = k;
    for (;;) {
      hist[t] = 0;
      __syncthreads();
      for (int64_t base = 0; base < len; base += kLongThreads) {  // block-uniform trip count: whole warps below
        const int64_t i = base + t;
        int digit = -1;
        if (i < len) {
          const u128 key = long_key(w, B, b, seg[lo + i]);
          if ((key >> (s + 8)) == (prefix >> (s + 8))) digit = (int)((unsigned)(key >> s) & 255u);
        }
        const unsigned peers = __match_any_sync(kFull, digit);
        if (digit >= 0 && lane == __ffs(peers) - 1) atomicAdd(&hist[digit], __popc(peers));
      }
      __syncthreads();
      // exclusive scan of the 256 bins; the thread whose bin holds the want-th key publishes it
      const int c = hist[t];
      int incl = c;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int o = __shfl_up_sync(kFull, incl, off);
        if (lane >= off) incl += o;
      }
      __syncthreads();  // every hist[t] read before the warp totals overwrite hist[0 .. 7]
      if (lane == 31) hist[wid] = incl;
      __syncthreads();
      int ex = incl - c;
      for (int i = 0; i < wid; ++i) ex += hist[i];
      if (ex < want && want <= ex + c) { sel_bin = t; sel_below = ex; sel_cnt = c; }
      __syncthreads();
      prefix |= (u128)sel_bin << s;
      want -= sel_below;
      if (sel_cnt == want) break;  // (at s = 0 a bin holds one key, so the loop ends there at the latest)
      s -= 8;
    }
    // the winners: every key whose digits down to s are at most the prefix's, exactly k of them
    if (t == 0) n_win = 0;
    __syncthreads();
    const u128 bound = prefix >> s;
    for (int64_t i = t; i < len; i += kLongThreads) {
      const int v = seg[lo + i];
      const u128 key = long_key(w, B, b, v);
      if ((key >> s) <= bound) {
        const int p = atomicAdd(&n_win, 1);
        sd[p] = (unsigned long long)(key >> 32);
        sv[p] = v;
      }
    }
    m = k;
  }
  int len2 = 32;
  while (len2 < m) len2 <<= 1;
  for (int i = m + t; i < len2; i += kLongThreads) { sd[i] = kUnreached; sv[i] = 0x7fffffff; }
  __syncthreads();
  long_sort(sd, sv, len2);
  int32_t* oi = out_idx + (s0 - row0 + b) * (int64_t)k;
  float* ol = out_len + (s0 - row0 + b) * (int64_t)k;
  for (int j = t; j < k; j += kLongThreads) {
    const bool found = j < m;
    oi[j] = found ? sv[j] : -1;
    ol[j] = found ? (float)__longlong_as_double((long long)sd[j]) : __int_as_float(0x7f800000);
  }
}

__global__ void path_reset_kernel(PathWs w, int64_t B) {
  const unsigned long long nt = w.ctr->touched;
  for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < nt;
       i += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t e = w.touched[i];
    const int64_t idx = (int64_t)(e >> 32) * B + (int64_t)(e & 0xffffffffull);
    w.dist[idx] = kUnreached;
    w.stamp[idx] = 0;
  }
}

// Runs the batches of [s_begin, s_end).  `finish(s0, nsrc)` enqueues the per-batch emission / selection and MUST
// leave the tile reset.  Blocking: one read of the queue length every kRoundsPerCheck rounds, at most n rounds.
template <class Finish>
int run_batches(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n, int64_t s_begin,
                int64_t s_end, double max_len, const PathWs& w, int64_t B, cudaStream_t st, Finish finish) {
  MDE_CUDA_TRY(cudaMemsetAsync(w.dist, 0xff, (size_t)(n * B) * sizeof(unsigned long long), st));
  MDE_CUDA_TRY(cudaMemsetAsync(w.stamp, 0, (size_t)(n * B) * sizeof(int), st));
  unsigned long long* pending = nullptr;
  MDE_CUDA_TRY(cudaMallocHost(&pending, sizeof(unsigned long long)));
  int rc = 0;
  for (int64_t s0 = s_begin; s0 < s_end && !rc; s0 += B) {
    const int nsrc = (int)((s_end - s0) < B ? (s_end - s0) : B);
    sssp_seed_kernel<<<(nsrc + 255) / 256, 256, 0, st>>>(w, B, s0, nsrc);
    ++g_launch_count;
    for (int64_t r = 1; r <= n; ++r) {
      sssp_relax_kernel<<<kRelaxBlocks, kRelaxThreads, 0, st>>>(indptr, indices, weights, w, B, max_len, (int)r);
      ++g_launch_count;
      if (r % kRoundsPerCheck != 0 && r != n) continue;
      cudaError_t err = cudaMemcpyAsync(pending, &w.ctr->queue[(r + 1) % 3], sizeof(unsigned long long),
                                        cudaMemcpyDeviceToHost, st);
      if (err == cudaSuccess) err = cudaStreamSynchronize(st);
      if (err != cudaSuccess) { rc = (int)err; break; }
      if (*pending == 0ull) break;  // no entry improved in the last round: the batch has converged
    }
    if (!rc) rc = finish(s0, nsrc);
  }
  cudaFreeHost(pending);
  if (!rc) { cudaError_t e = cudaStreamSynchronize(st); if (e == cudaSuccess) e = cudaPeekAtLastError(); rc = (int)e; }
  return rc;
}

inline double length_limit(double max_length) {
  return (max_length > 0.0 && max_length < INFINITY) ? max_length : INFINITY;
}

// k-NN lists of the sources [s_begin, s_end) into output rows 0 .. s_end - s_begin - 1.  Every list is a function of
// its source alone (the lengths are the schedule-free fixed point, ties break by node index), so it does not depend
// on the batch size or on where the batches start.  `long_select`: knn_select_long_kernel instead of knn_select_kernel.
int graph_knn_range(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n, int64_t s_begin,
                    int64_t s_end, int k, double max_distance, int32_t* out_idx, float* out_len, void* ws,
                    int64_t ws_bytes, bool long_select, cudaStream_t st) {
  const int64_t B = path_batch(n, s_end - s_begin, ws_bytes);
  const PathWs w = path_ws(ws, n, B);
  return run_batches(indptr, indices, weights, n, s_begin, s_end, length_limit(max_distance), w, B, st,
                     [&](int64_t s0, int nsrc) -> int {
                       MDE_CUDA_TRY(cudaMemsetAsync(w.seg_count, 0, (size_t)B * sizeof(int), st));
                       knn_count_kernel<<<kRelaxBlocks, 256, 0, st>>>(w, s0);
                       knn_scan_kernel<<<1, 1024, 0, st>>>(w, (int)B);
                       knn_scatter_kernel<<<kRelaxBlocks, 256, 0, st>>>(w, s0);
                       if (long_select)
                         knn_select_long_kernel<<<nsrc, kLongThreads, 0, st>>>(w, B, s0, s_begin, k, out_idx,
                                                                              out_len);
                       else
                         knn_select_kernel<<<(nsrc * 32 + 255) / 256, 256, 0, st>>>(w, B, s0, s_begin, nsrc, k,
                                                                                    out_idx, out_len);
                       path_reset_kernel<<<kRelaxBlocks, 256, 0, st>>>(w, B);
                       g_launch_count += 5;
                       return 0;
                     });
}

}  // namespace

extern "C" {

int64_t mde_graph_hops_ws_bytes(int64_t n) { return 3 * n * kWords * (int64_t)sizeof(uint64_t) + 64; }

int64_t mde_graph_sssp_ws_bytes(int64_t n, int batch) {
  if (n < 1 || batch < 32 || batch % 32) return -1;
  return path_ws_bytes(n, batch);
}

int64_t mde_graph_knn_ws_bytes(int64_t n, int batch) { return mde_graph_sssp_ws_bytes(n, batch); }

int mde_graph_knn_max_k(void) { return kKnnMaxK; }

int mde_graph_sssp(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n, int64_t s_begin,
                   int64_t s_end, double max_length, double retain, uint64_t seed, int32_t* out_src,
                   int32_t* out_dst, float* out_len, int64_t cap, unsigned long long* count_dev, void* ws,
                   int64_t ws_bytes, void* stream) {
  if (!indptr || !indices || n < 1 || n >= (1ll << 31) || s_begin < 0 || s_end > n || s_begin > s_end ||
      !count_dev || !ws || cap < 0 || (cap > 0 && (!out_src || !out_dst || !out_len)))
    return MDE_E_INVALID;
  const int64_t B = path_batch(n, s_end - s_begin, ws_bytes);
  if (B < 32) return MDE_E_INVALID;
  if (s_begin == s_end) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  const PathWs w = path_ws(ws, n, B);
  const uint64_t thresh = (retain >= 1.0) ? ~0ull : (uint64_t)(retain * 18446744073709551616.0);
  return run_batches(indptr, indices, weights, n, s_begin, s_end, length_limit(max_length), w, B, st,
                     [&](int64_t s0, int) -> int {
                       sssp_emit_reset_kernel<<<kRelaxBlocks, 256, 0, st>>>(w, B, n, s0, seed, thresh, out_src,
                                                                            out_dst, out_len, cap, count_dev);
                       ++g_launch_count;
                       return 0;
                     });
}

int mde_graph_knn(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n, int k,
                  double max_distance, int32_t* out_idx, float* out_len, void* ws, int64_t ws_bytes, void* stream) {
  if (!indptr || !indices || n < 1 || n >= (1ll << 31) || k < 1 || k > kKnnMaxK || !out_idx || !out_len || !ws)
    return MDE_E_INVALID;
  if (path_batch(n, n, ws_bytes) < 32) return MDE_E_INVALID;
  return graph_knn_range(indptr, indices, weights, n, 0, n, k, max_distance, out_idx, out_len, ws, ws_bytes, false,
                         (cudaStream_t)stream);
}

int mde_graph_knn_rows(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n,
                       int64_t s_begin, int64_t s_end, int k, double max_distance, int32_t* out_idx, float* out_len,
                       void* ws, int64_t ws_bytes, void* stream) {
  if (!indptr || !indices || n < 1 || n >= (1ll << 31) || s_begin < 0 || s_end > n || s_begin > s_end || k < 1 ||
      k > kKnnMaxK || !out_idx || !out_len || !ws || ws_bytes < path_ws_bytes(n, 32))
    return MDE_E_INVALID;
  if (s_begin == s_end) return 0;
  return graph_knn_range(indptr, indices, weights, n, s_begin, s_end, k, max_distance, out_idx, out_len, ws,
                         ws_bytes, false, (cudaStream_t)stream);
}

int mde_graph_knn_long_max_k(void) { return kKnnLongMaxK; }

int mde_graph_knn_long(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n, int k,
                       double max_distance, int32_t* out_idx, float* out_len, void* ws, int64_t ws_bytes,
                       void* stream) {
  if (!indptr || !indices || n < 1 || n >= (1ll << 31) || k < 1 || k > kKnnLongMaxK || !out_idx || !out_len || !ws)
    return MDE_E_INVALID;
  if (path_batch(n, n, ws_bytes) < 32) return MDE_E_INVALID;
  return graph_knn_range(indptr, indices, weights, n, 0, n, k, max_distance, out_idx, out_len, ws, ws_bytes, true,
                         (cudaStream_t)stream);
}

int mde_graph_knn_long_rows(const int32_t* indptr, const int32_t* indices, const float* weights, int64_t n,
                            int64_t s_begin, int64_t s_end, int k, double max_distance, int32_t* out_idx,
                            float* out_len, void* ws, int64_t ws_bytes, void* stream) {
  if (!indptr || !indices || n < 1 || n >= (1ll << 31) || s_begin < 0 || s_end > n || s_begin > s_end || k < 1 ||
      k > kKnnLongMaxK || !out_idx || !out_len || !ws || ws_bytes < path_ws_bytes(n, 32))
    return MDE_E_INVALID;
  if (s_begin == s_end) return 0;
  return graph_knn_range(indptr, indices, weights, n, s_begin, s_end, k, max_distance, out_idx, out_len, ws,
                         ws_bytes, true, (cudaStream_t)stream);
}

int mde_graph_hops(const int32_t* indptr, const int32_t* indices, int64_t n, int64_t s_begin, int64_t s_end,
                   int max_length, double retain, uint64_t seed, int32_t* out_src, int32_t* out_dst,
                   float* out_len, int64_t cap, unsigned long long* count_dev, void* ws, int64_t ws_bytes,
                   void* stream) {
  if (!indptr || !indices || n < 1 || s_begin < 0 || s_end > n || s_begin > s_end || !count_dev || !ws ||
      ws_bytes < mde_graph_hops_ws_bytes(n) || n >= (1ll << 31) || (cap > 0 && (!out_src || !out_dst || !out_len)))
    return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  uint64_t* visited = reinterpret_cast<uint64_t*>(ws);
  uint64_t* fa = visited + n * kWords;
  uint64_t* fb = fa + n * kWords;
  int* any_d = reinterpret_cast<int*>(fb + n * kWords);
  const uint64_t thresh = (retain >= 1.0) ? ~0ull : (uint64_t)(retain * 18446744073709551616.0);
  const int limit = (max_length <= 0) ? 0x7fffffff : max_length;
  const int tb = 256;
  const int nb = ceil_div_i64(n * kWords, tb);
  int* any_h = nullptr;
  MDE_CUDA_TRY(cudaMallocHost(&any_h, sizeof(int)));
  int rc = 0;
  for (int64_t s0 = s_begin; s0 < s_end && !rc; s0 += kBatch) {
    const int nsrc = (int)((s_end - s0) < kBatch ? (s_end - s0) : kBatch);
    hops_init_kernel<<<nb, tb, 0, st>>>(visited, fa, n, s0, nsrc);
    ++g_launch_count;
    uint64_t *fin = fa, *fout = fb;
    for (int level = 1; level <= limit; ++level) {
      cudaError_t err = cudaMemsetAsync(any_d, 0, sizeof(int), st);
      if (err != cudaSuccess) { rc = (int)err; break; }
      hops_level_kernel<<<nb, tb, 0, st>>>(indptr, indices, fin, visited, fout, n, s0, level, 1, seed, thresh, out_src,
                                          out_dst, out_len, cap, count_dev, any_d);
      ++g_launch_count;
      err = cudaMemcpyAsync(any_h, any_d, sizeof(int), cudaMemcpyDeviceToHost, st);
      if (err == cudaSuccess) err = cudaStreamSynchronize(st);
      if (err != cudaSuccess) { rc = (int)err; break; }
      if (!*any_h) break;  // every search of the batch has stopped growing
      uint64_t* tmp = fin; fin = fout; fout = tmp;
    }
  }
  cudaFreeHost(any_h);
  if (!rc) { cudaError_t e = cudaPeekAtLastError(); if (e != cudaSuccess) rc = (int)e; }
  return rc;
}

}  // extern "C"
