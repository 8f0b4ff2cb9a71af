// mde_knn_graph.cu -- neighbour lists to a weighted undirected edge list on the device: the edges and weights that
// Graph.from_edges(pairs, None, n) followed by .edges / .weights gives for the directed pairs (i, idx[i][s]).
//
// The pair {a, b}, a < b, is listed by a (a -> b) and/or by b (b -> a).  Row a owns it: its candidates are
//
//   F_a   the entries of row a that are > a (forward list), and
//   R_a   the rows u > a whose list holds a (reverse list),
//
// and its output is the distinct values of F_a u R_a in ascending order, each weighted by its number of occurrences
// in both lists (scipy sums the duplicates).  The call is
//
//   prep       one warp per row: check the entries, bitonic-sort the row's entries > i (P per lane: 2 for k <= 64,
//              8 for k <= 256), keep each distinct value once with its multiplicity (F_i, acount[i] values), and
//              write the reverse sort's input (key = v for an entry u -> v with v < u, else n; value = u)
//   sort       one stable CUB radix sort of (key, value) over ceil(log2(n + 1)) bits: R_v = the rows u > v that list
//              v, ascending, at [rev_off[v], rev_off[v + 1]) (rev_off by binary search)
//   flags      per reverse entry p: 1 when it is the first of its run of equal u in R_v and u is not in F_v (binary
//              search in <= k values); an exclusive scan gives S_R
//   offsets    cnt[i] = acount[i] + (R-only runs of row i), scanned into row_off
//
// and the emit pass writes every output at its rank in the union, without atomics:
//
//   F value a at slot r:      row_off[i] + r + (R-only runs of R_i below a),      weight mult + (count of a in R_i)
//   R-only run of u at p:     row_off[v] + (R-only runs before p) + (values of F_v below u),   weight its run length
//
// Every step is element-parallel (one thread per entry, binary searches into the lists), so a row that every other
// row lists (a hub, |R_v| up to n - 1) costs no more than its entries.  The result is a function of (idx, n, k)
// alone: everything read is written by the call first, and nothing depends on the order threads run.
#include <cuda_runtime.h>
#include <cub/cub.cuh>

#include <climits>
#include <cstdint>

#include "mde_common.cuh"

using namespace mde;

namespace {

constexpr int kMaxK = 64;       // mde_knn_graph_*: the prep pass sorts 2 entries per lane
constexpr int kLongMaxK = 256;  // mde_knn_graph_*_long: 8 entries per lane
constexpr int kSentinel = INT_MAX;  // past every valid value: sorts last

int bits_for(int64_t count) {  // smallest b with 2^b >= count
  int b = 0;
  while (b < 62 && (1ll << b) < count) ++b;
  return b;
}

// Workspace layout (host arithmetic only).  The sort runs on CUB double buffers; whichever buffer of each pair does
// not hold the sorted result is reused for the scan's input (flags) and output (S_R), so both are N + 1 long.
struct GraphLayout {
  int64_t N;  // n * k
  size_t off_hdr, off_acount, off_fwd, off_fmul, off_k0, off_k1, off_v0, off_v1, off_rev, off_cnt, off_row, off_tmp;
  size_t tmp_bytes, total;
};

GraphLayout graph_layout(int64_t n, int k) {
  GraphLayout L;
  L.N = n * k;
  // CUB's scratch for a double-buffer radix sort and for the scans: bin counts and look-back state, well under a
  // byte per item; the call checks CUB's exact figure against this bound (MDE_E_ALLOC should it ever be short)
  L.tmp_bytes = (size_t)(L.N + n) / 2 + (16u << 20);
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  const size_t items = (size_t)L.N + 1;
  size_t o = 0;
  L.off_hdr = o; o = up(o + 16);                       // {flag, total, sort buffer}
  L.off_acount = o; o = up(o + (size_t)n * 4);
  L.off_fwd = o; o = up(o + (size_t)L.N * 4);
  L.off_fmul = o; o = up(o + (size_t)L.N);           // multiplicity - 1 (1 .. 256 fits a byte)
  L.off_k0 = o; o = up(o + items * 4);
  L.off_k1 = o; o = up(o + items * 4);
  L.off_v0 = o; o = up(o + items * 4);
  L.off_v1 = o; o = up(o + items * 4);
  L.off_rev = o; o = up(o + (size_t)(n + 1) * 4);
  L.off_cnt = o; o = up(o + (size_t)(n + 1) * 4);
  L.off_row = o; o = up(o + (size_t)(n + 1) * 4);
  L.off_tmp = o; o = up(o + L.tmp_bytes);
  L.total = o;
  return L;
}

// The buffers of one call.  The sort runs from (k0, v0); CUB says which buffer of each pair it ends in.
struct GraphBufs {
  int32_t* hdr;  // {flag, total, 1 when the sorted entries are in (k1, v1)}
  int32_t* acount;
  int32_t* fwd;
  uint8_t* fmul;
  int32_t *k0, *k1, *v0, *v1;
  int32_t *rev_off, *cnt, *row_off;
  void* tmp;
};

GraphBufs carve(uint8_t* w, const GraphLayout& L) {
  auto at = [w](size_t off) { return reinterpret_cast<int32_t*>(w + off); };
  GraphBufs B;
  B.hdr = at(L.off_hdr);
  B.acount = at(L.off_acount);
  B.fwd = at(L.off_fwd);
  B.fmul = w + L.off_fmul;
  B.k0 = at(L.off_k0); B.k1 = at(L.off_k1);
  B.v0 = at(L.off_v0); B.v1 = at(L.off_v1);
  B.rev_off = at(L.off_rev);
  B.cnt = at(L.off_cnt);
  B.row_off = at(L.off_row);
  B.tmp = w + L.off_tmp;
  return B;
}

// First index in a[lo, hi) whose value is >= x (strict: > x).
template <bool kStrict>
__device__ __forceinline__ int32_t search(const int32_t* __restrict__ a, int32_t lo, int32_t hi, int32_t x) {
  while (lo < hi) {
    const int32_t mid = lo + ((hi - lo) >> 1);
    const int32_t y = __ldg(a + mid);
    if (kStrict ? y <= x : y < x) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// One warp per row of k <= 32 P entries: the check, the forward list and the reverse sort's input.
template <int P>
__global__ void __launch_bounds__(256)
knn_graph_prep_kernel(const int32_t* __restrict__ idx, int64_t n, int k, int32_t* __restrict__ flag,
                      int32_t* __restrict__ acount, int32_t* __restrict__ fwd, uint8_t* __restrict__ fmul,
                      int32_t* __restrict__ rkey, int32_t* __restrict__ rval) {
  constexpr int kSlots = 32 * P;
  const int lane = threadIdx.x & 31;
  const int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (i >= n) return;
  const int32_t* row = idx + i * k;
  int32_t v[P];
  bool bad = false;
#pragma unroll
  for (int h = 0; h < P; ++h) {
    const int e = lane + 32 * h;
    const int32_t x = e < k ? __ldg(row + e) : -1;
    bad |= x == i || x < -1 || x >= n;
    v[h] = (x > i && x < n) ? x : kSentinel;
    if (e < k) {
      rkey[i * k + e] = (x >= 0 && x < i) ? x : (int32_t)n;
      rval[i * k + e] = (int32_t)i;
    }
  }
  if (__any_sync(kFull, bad) && lane == 0) *flag = 1;
  // bitonic sort of the kSlots slots e = lane + 32 h, ascending (strides >= 32 pair registers of one lane)
#pragma unroll
  for (int size = 2; size <= kSlots; size <<= 1) {
#pragma unroll
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      int32_t o[P];
#pragma unroll
      for (int h = 0; h < P; ++h) o[h] = stride >= 32 ? v[h ^ (stride >> 5)] : __shfl_xor_sync(kFull, v[h], stride);
#pragma unroll
      for (int h = 0; h < P; ++h) {
        const int e = lane + 32 * h;
        const bool asc = (e & size) == 0, lower = (e & stride) == 0;
        v[h] = (lower == asc) ? min(v[h], o[h]) : max(v[h], o[h]);
      }
    }
  }
  // distinct values with their multiplicities, compacted to the front of the row; H[h] / V[h]: the heads / valid
  // values among the slots lane + 32 h
  uint32_t H[P], V[P];
  bool head[P];
#pragma unroll
  for (int h = 0; h < P; ++h) {
    const int32_t up = __shfl_up_sync(kFull, v[h], 1);
    const int32_t last = h ? __shfl_sync(kFull, v[h ? h - 1 : 0], 31) : INT_MIN;
    const int32_t prev = lane ? up : last;
    const bool valid = v[h] != kSentinel;
    head[h] = valid && prev != v[h];
    H[h] = __ballot_sync(kFull, head[h]);
    V[h] = __ballot_sync(kFull, valid);
  }
  int nvalid = 0, heads = 0;  // the valid values are a prefix
#pragma unroll
  for (int h = 0; h < P; ++h) { nvalid += __popc(V[h]); heads += __popc(H[h]); }
  int below = 0;  // heads in the registers before h
#pragma unroll
  for (int h = 0; h < P; ++h) {
    if (head[h]) {
      const int e = lane + 32 * h;
      int next = nvalid;  // the slot of the next head, or the end of the valid values
      const uint32_t above = H[h] & ~((2u << lane) - 1);  // (2u << 31 wraps to 0: nothing above lane 31)
      if (above) {
        next = 32 * h + __ffs(above) - 1;
      } else {
#pragma unroll
        for (int h2 = P - 1; h2 > h; --h2) if (H[h2]) next = 32 * h2 + __ffs(H[h2]) - 1;
      }
      const int r = below + __popc(H[h] & ((1u << lane) - 1));
      fwd[i * k + r] = v[h];
      fmul[i * k + r] = (uint8_t)(next - e - 1);
    }
    below += __popc(H[h]);
  }
  if (lane == 0) acount[i] = heads;
}

// rev_off[v] = first p with key[p] >= v, for v in [0, n] (a binary search each: long runs of one key, or keys that
// never occur, cost nothing extra).
__global__ void knn_graph_rev_off_kernel(const int32_t* __restrict__ key, int64_t N, int64_t n,
                                         int32_t* __restrict__ rev_off) {
  const int64_t v = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (v > n) return;
  rev_off[v] = search<false>(key, 0, (int32_t)N, (int32_t)v);
}

// 1 where a reverse entry starts a run of equal rows and that row is not in the owner's forward list; 0 elsewhere,
// including the entries with key n past rev_off[n] and the extra item N.
__global__ void knn_graph_flag_kernel(const int32_t* __restrict__ key, const int32_t* __restrict__ val, int64_t N,
                                      int k, const int32_t* __restrict__ rev_off, const int32_t* __restrict__ acount,
                                      const int32_t* __restrict__ fwd, int64_t n, int32_t* __restrict__ flag_out) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p > N) return;
  int32_t f = 0;
  if (p < rev_off[n]) {
    const int32_t v = key[p], u = val[p];
    if (p == rev_off[v] || val[p - 1] != u) {
      const int32_t* F = fwd + (int64_t)v * k;
      const int32_t a = acount[v];
      const int32_t s = search<false>(F, 0, a, u);
      f = !(s < a && F[s] == u);
    }
  }
  flag_out[p] = f;
}

__global__ void knn_graph_count_kernel(int64_t n, const int32_t* __restrict__ acount,
                                       const int32_t* __restrict__ rev_off, const int32_t* __restrict__ S,
                                       int32_t* __restrict__ cnt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  cnt[i] = i < n ? acount[i] + S[rev_off[i + 1]] - S[rev_off[i]] : 0;
}

// The sorted reverse entries and S_R as the count call left them; hdr[2] says which buffer of each pair holds them.
struct Sorted {
  const int32_t* hdr;
  const int32_t *k0, *k1, *v0, *v1;
  __device__ __forceinline__ void get(const int32_t*& key, const int32_t*& val, const int32_t*& S) const {
    const bool sel = hdr[2] != 0;
    key = sel ? k1 : k0;
    val = sel ? v1 : v0;
    S = sel ? v0 : v1;  // the scan's output went to the values' free buffer
  }
};

// The forward values of every row at their ranks in the union (one thread per slot).
__global__ void knn_graph_emit_fwd_kernel(int64_t n, int k, const int32_t* __restrict__ acount,
                                          const int32_t* __restrict__ fwd, const uint8_t* __restrict__ fmul,
                                          Sorted sorted, const int32_t* __restrict__ rev_off,
                                          const int32_t* __restrict__ row_off, int64_t* __restrict__ edges,
                                          float* __restrict__ weights) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n * k) return;
  const int64_t i = t / k;
  const int r = (int)(t - i * k);
  if (r >= acount[i]) return;
  const int32_t *rkey, *rval, *S;
  sorted.get(rkey, rval, S);
  const int32_t a = fwd[t];
  const int32_t lo = rev_off[i], hi = rev_off[i + 1];
  const int32_t lb = search<false>(rval, lo, hi, a), ub = search<true>(rval, lb, hi, a);
  const int64_t pos = (int64_t)row_off[i] + r + (S[lb] - S[lo]);
  edges[2 * pos] = i;
  edges[2 * pos + 1] = a;
  weights[pos] = (float)(fmul[t] + 1 + (ub - lb));
}

// The runs of reverse entries whose row is not in the owner's forward list (one thread per reverse entry).
__global__ void knn_graph_emit_rev_kernel(int64_t N, int k, Sorted sorted, const int32_t* __restrict__ acount,
                                          const int32_t* __restrict__ fwd, const int32_t* __restrict__ rev_off,
                                          const int32_t* __restrict__ row_off, int64_t n, int64_t* __restrict__ edges,
                                          float* __restrict__ weights) {
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N || p >= rev_off[n]) return;
  const int32_t *key, *val, *S;
  sorted.get(key, val, S);
  if (S[p + 1] == S[p]) return;  // not an R-only run head
  const int32_t v = key[p], u = val[p];
  const int32_t lo = rev_off[v], hi = rev_off[v + 1];
  const int32_t ub = search<true>(val, (int32_t)p + 1, hi, u);
  const int32_t below = search<false>(fwd + (int64_t)v * k, 0, acount[v], u);
  const int64_t pos = (int64_t)row_off[v] + (S[p] - S[lo]) + below;
  edges[2 * pos] = v;
  edges[2 * pos + 1] = u;
  weights[pos] = (float)(ub - (int32_t)p);
}

// Header: {flag, total, which buffer of each sort pair holds the sorted entries}.
__global__ void knn_graph_total_kernel(const int32_t* __restrict__ row_off, int64_t n, int sel,
                                       int32_t* __restrict__ hdr) {
  hdr[1] = row_off[n];
  hdr[2] = sel;
}

unsigned grid_for(int64_t threads) { return (unsigned)((threads + 255) / 256); }

// CUB's scratch for the sort and the two scans (a query: no device work).
int graph_cub_bytes(int64_t n, int64_t N, size_t* bytes) {
  size_t t1 = 0, t2 = 0, t3 = 0;
  cub::DoubleBuffer<int32_t> kb(nullptr, nullptr), vb(nullptr, nullptr);
  MDE_CUDA_TRY(cub::DeviceRadixSort::SortPairs(nullptr, t1, kb, vb, (int64_t)N, 0, bits_for(n + 1)));
  MDE_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t2, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(N + 1)));
  MDE_CUDA_TRY(cub::DeviceScan::ExclusiveSum(nullptr, t3, (const int32_t*)nullptr, (int32_t*)nullptr, (int)(n + 1)));
  *bytes = t1 > t2 ? t1 : t2;
  if (t3 > *bytes) *bytes = t3;
  return 0;
}

bool bad_args(int64_t n, int k, int max_k) { return n < 1 || k < 1 || k > max_k; }

// The checks both calls share: every one of them is host arithmetic.
int check_ws(int64_t n, int k, const void* ws, size_t ws_bytes, GraphLayout* L) {
  if (n * k >= INT_MAX) return MDE_E_UNSUPPORTED;
  *L = graph_layout(n, k);
  if (ws_bytes < L->total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  return 0;
}

// The calls of both entry families; max_k is the family's bound on k.
int graph_ws_bytes(int64_t n, int k, int max_k, size_t* bytes) {
  if (!bytes || bad_args(n, k, max_k)) return MDE_E_INVALID;
  if (n * k >= INT_MAX) return MDE_E_UNSUPPORTED;
  *bytes = graph_layout(n, k).total;
  return 0;
}

int graph_count(const int32_t* idx, int64_t n, int k, int max_k, void* ws, size_t ws_bytes, int64_t* count,
                void* stream) {
  if (!idx || !ws || !count || bad_args(n, k, max_k)) return MDE_E_INVALID;
  GraphLayout L;
  int rc = check_ws(n, k, ws, ws_bytes, &L);
  if (rc) return rc;
  size_t cub_bytes = 0;
  if ((rc = graph_cub_bytes(n, L.N, &cub_bytes))) return rc;
  if (cub_bytes > L.tmp_bytes) return MDE_E_ALLOC;
  cudaStream_t st = (cudaStream_t)stream;
  uint8_t* w = static_cast<uint8_t*>(ws);
  const GraphBufs B = carve(w, L);
  MDE_CUDA_TRY(cudaMemsetAsync(B.hdr, 0, 16, st));
  if (k <= kMaxK)
    knn_graph_prep_kernel<2><<<grid_for(n * 32), 256, 0, st>>>(idx, n, k, B.hdr, B.acount, B.fwd, B.fmul, B.k0, B.v0);
  else
    knn_graph_prep_kernel<8><<<grid_for(n * 32), 256, 0, st>>>(idx, n, k, B.hdr, B.acount, B.fwd, B.fmul, B.k0, B.v0);
  MDE_LAUNCH_CHECK();
  cub::DoubleBuffer<int32_t> kb(B.k0, B.k1), vb(B.v0, B.v1);
  size_t tb = L.tmp_bytes;
  MDE_CUDA_TRY(cub::DeviceRadixSort::SortPairs(B.tmp, tb, kb, vb, (int64_t)L.N, 0, bits_for(n + 1), st));
  // the sorted entries are in kb / vb.Current(); their Alternate() buffers take the run flags and S_R
  knn_graph_rev_off_kernel<<<grid_for(n + 1), 256, 0, st>>>(kb.Current(), L.N, n, B.rev_off);
  MDE_LAUNCH_CHECK();
  knn_graph_flag_kernel<<<grid_for(L.N + 1), 256, 0, st>>>(kb.Current(), vb.Current(), L.N, k, B.rev_off, B.acount,
                                                           B.fwd, n, kb.Alternate());
  MDE_LAUNCH_CHECK();
  tb = L.tmp_bytes;
  MDE_CUDA_TRY(cub::DeviceScan::ExclusiveSum(B.tmp, tb, kb.Alternate(), vb.Alternate(), (int)(L.N + 1), st));
  knn_graph_count_kernel<<<grid_for(n + 1), 256, 0, st>>>(n, B.acount, B.rev_off, vb.Alternate(), B.cnt);
  MDE_LAUNCH_CHECK();
  tb = L.tmp_bytes;
  MDE_CUDA_TRY(cub::DeviceScan::ExclusiveSum(B.tmp, tb, B.cnt, B.row_off, (int)(n + 1), st));
  knn_graph_total_kernel<<<1, 1, 0, st>>>(B.row_off, n, kb.Current() == B.k1 ? 1 : 0, B.hdr);
  MDE_LAUNCH_CHECK();
  int32_t h[2] = {0, 0};
  MDE_CUDA_TRY(cudaMemcpyAsync(h, B.hdr, sizeof(h), cudaMemcpyDeviceToHost, st));
  MDE_CUDA_TRY(cudaStreamSynchronize(st));
  if (h[0]) return MDE_E_INVALID;
  *count = h[1];
  return 0;
}

int graph_emit(int64_t n, int k, int max_k, const void* ws, size_t ws_bytes, int64_t* edges_out, float* weights_out,
               void* stream) {
  if (!ws || !edges_out || !weights_out || bad_args(n, k, max_k)) return MDE_E_INVALID;
  GraphLayout L;
  const int rc = check_ws(n, k, ws, ws_bytes, &L);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const GraphBufs B = carve(const_cast<uint8_t*>(static_cast<const uint8_t*>(ws)), L);
  const Sorted sorted{B.hdr, B.k0, B.k1, B.v0, B.v1};
  knn_graph_emit_fwd_kernel<<<grid_for(L.N), 256, 0, st>>>(n, k, B.acount, B.fwd, B.fmul, sorted, B.rev_off,
                                                           B.row_off, edges_out, weights_out);
  MDE_LAUNCH_CHECK();
  knn_graph_emit_rev_kernel<<<grid_for(L.N), 256, 0, st>>>(L.N, k, sorted, B.acount, B.fwd, B.rev_off, B.row_off, n,
                                                           edges_out, weights_out);
  MDE_LAUNCH_CHECK();
  return 0;
}

}  // namespace

extern "C" {

int mde_knn_graph_max_k(void) { return kMaxK; }

int mde_knn_graph_ws_bytes(int64_t n, int k, size_t* bytes) { return graph_ws_bytes(n, k, kMaxK, bytes); }

int mde_knn_graph_count(const int32_t* idx, int64_t n, int k, void* ws, size_t ws_bytes, int64_t* count,
                        void* stream) {
  return graph_count(idx, n, k, kMaxK, ws, ws_bytes, count, stream);
}

int mde_knn_graph_emit(int64_t n, int k, const void* ws, size_t ws_bytes, int64_t* edges_out, float* weights_out,
                       void* stream) {
  return graph_emit(n, k, kMaxK, ws, ws_bytes, edges_out, weights_out, stream);
}

int mde_knn_graph_long_max_k(void) { return kLongMaxK; }

int mde_knn_graph_long_ws_bytes(int64_t n, int k, size_t* bytes) { return graph_ws_bytes(n, k, kLongMaxK, bytes); }

int mde_knn_graph_long_count(const int32_t* idx, int64_t n, int k, void* ws, size_t ws_bytes, int64_t* count,
                             void* stream) {
  return graph_count(idx, n, k, kLongMaxK, ws, ws_bytes, count, stream);
}

int mde_knn_graph_long_emit(int64_t n, int k, const void* ws, size_t ws_bytes, int64_t* edges_out,
                            float* weights_out, void* stream) {
  return graph_emit(n, k, kLongMaxK, ws, ws_bytes, edges_out, weights_out, stream);
}

}  // extern "C"
