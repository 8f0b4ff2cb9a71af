// mde_knn.cu -- exact k-nearest neighbours of the rows of a data matrix (SURVEY section 8 row f3).
//
// Replaces the neighbour search of pymde/preprocess/data_matrix.py:91-178 (scikit-learn brute force below 10 000
// rows, pynndescent above) by an exact search whose cross terms run on the Hopper tensor cores (wgmma):
//
//   prep     X (n x d fp32) -> Xh, Xl (n_pad x K_pad bf16, x = hi + lo to 2^-16), ||x||^2 (fp32; +inf on padding)
//   tiles    one CTA per 128 query rows sweeps ALL candidates in tiles of 128:
//              a producer warp stages 64-wide K blocks of the hi and lo parts of both operands in shared memory with
//              TMA (cp.async.bulk.tensor.2d, 128-byte swizzle; 2 stages x 64 KB, mbarrier pipeline), and two consumer
//              warpgroups (64 query rows each) issue
//              wgmma.mma_async.m64n128k16.f32.bf16.bf16  D[64 x 128] += Ah Bh^T + Ah Bl^T + Al Bh^T   (fp32 registers),
//              stage the finished accumulator in shared memory, form ||x||^2 - 2 q.x and keep, per query row, the
//              KK = 32 smallest in thread-private lists (two threads per row, merged at the end).  The n x n distance
//              matrix never exists.
//   re-rank  exact fp32 sum (q - x)^2 of the KK candidates of a row (one warp per row), k smallest, ascending.
//
// The bf16 x 3 split leaves an error of ~2^-16 |q||x| on a cross term, far below the gap between the k-th and the
// (k + 8)-th neighbour of real data, and the re-rank removes it from the result: the neighbour lists are those of a
// brute-force fp32 search (ties and fp32 rounding aside).  k <= 24.
//
// Hangs are not an option on a shared GPU: every mbarrier wait is bounded (mde_tma.cuh) and traps.
#include <cuda.h>  // CUtensorMap and its enums (types only: the encoder is fetched with cudaGetDriverEntryPoint)
#include <cuda_bf16.h>

#include <cstdint>
#include <cstdlib>

#include "mde_common.cuh"
#include "mde_tma.cuh"

using namespace mde;

namespace {

constexpr int kTileM = 128;                 // query rows per CTA (two warpgroups of 64)
constexpr int kTileN = 128;                 // candidates per tile = wgmma N
constexpr int kBlockK = 64;                 // bf16 elements per 128-byte swizzle row
constexpr int kWgmmaK = 16;                 // K of one wgmma.m64n128k16
constexpr int kStages = 2;
constexpr int kKK = 32;                     // candidates kept per row before the exact re-rank
constexpr int kMaxK = 24;
constexpr int kRowBytes = kBlockK * 2;      // 128
constexpr int kOpBytes = 128 * kRowBytes;   // 16 KB: one 128-row operand block (hi or lo)
constexpr int kStageBytes = 4 * kOpBytes;   // A hi, A lo, B hi, B lo = 64 KB
constexpr int kConsumerWarps = 8;           // warps 0-7: two consumer warpgroups; warp 8: TMA producer
constexpr int kThreads = (kConsumerWarps + 1) * 32;
constexpr int kAccStride = kTileN + 2;      // floats per staged accumulator row: the scan's column reads are conflict-free
constexpr int kSmemBytes = kStages * kStageBytes + 1024 /* alignment slack */ + kTileM * kAccStride * 4 +
                           2 * kTileN * 4 /* norms */ + 64 /* barriers */;
static_assert(kTileM == 128 && kTileN == 128, "one TMA box (64 x 128) serves both operands");
static_assert(kSmemBytes <= 227 * 1024, "H100: at most 227 KB of shared memory per block");

// ---------------------------------------------------------------------------------------------------------------
// PTX wrappers (wgmma / tensor TMA); mbarriers come from mde_tma.cuh
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(x), "r"(y)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void named_bar_sync(int id, int count) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator registers across the asynchronous wgmma window
__device__ __forceinline__ void fence_operand(float& r) { asm volatile("" : "+f"(r)::"memory"); }

// D[64 x 128] (+)= A[smem, 64 x 16] * B[smem, 128 x 16]^T, both operands K-major; issued by the whole warpgroup.
// Accumulator fragment: d[4 j + {0, 1}] = (row 16 w + lane / 4, col 8 j + 2 (lane % 4) + {0, 1}), d[4 j + {2, 3}] the
// same columns of row + 8 (w = warp within the warpgroup).
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "setp.ne.b32 p, %66, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// Shared-memory matrix descriptor (sm_90 wgmma) of a K-major operand block staged by TMA with the 128-byte swizzle:
// rows of 128 bytes, 8-row groups 1024 bytes apart (stride byte offset), one swizzle atom along K (leading byte
// offset unused), layout type 1 = SWIZZLE_128B in bits 62-63.  Blocks start 1024-aligned (base offset 0).
__device__ __forceinline__ uint64_t smem_desc_sw128(uint32_t saddr) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | ((uint64_t)(1024u >> 4) << 32) | (1ull << 62);
}

// ---------------------------------------------------------------------------------------------------------------
// prep: bf16 hi / lo split (zero padded to n_pad x k_pad) and squared norms (+inf on padded rows)
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
knn_prep_kernel(const float* __restrict__ X, int64_t n, int d, int64_t n_pad, int k_pad, __nv_bfloat16* __restrict__ Xh,
                __nv_bfloat16* __restrict__ Xl, float* __restrict__ norms) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n_pad) return;
  float acc = 0.0f;
  for (int c = lane; c < k_pad; c += 32) {
    const float x = (row < n && c < d) ? X[row * d + c] : 0.0f;
    const __nv_bfloat16 h = __float2bfloat16_rn(x);
    const __nv_bfloat16 l = __float2bfloat16_rn(x - __bfloat162float(h));
    Xh[row * k_pad + c] = h;
    Xl[row * k_pad + c] = l;
    acc += x * x;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
  if (lane == 0) norms[row] = (row < n) ? acc : __int_as_float(0x7f800000);
}

// Replace the worst of the KK kept candidates by (dist, col) and find the new worst.  Static indices only, so the
// lists stay in registers.
__device__ __forceinline__ void keep_candidate(float (&bd)[kKK], int (&bi)[kKK], float dist, int col, float& thr,
                                               int& worst) {
#pragma unroll
  for (int q = 0; q < kKK; ++q) {
    if (q == worst) { bd[q] = dist; bi[q] = col; }
  }
  float m = bd[0]; int w = 0;
#pragma unroll
  for (int q = 1; q < kKK; ++q) { if (bd[q] > m) { m = bd[q]; w = q; } }
  thr = m; worst = w;
}

// ---------------------------------------------------------------------------------------------------------------
// tiles: tensor-core cross terms + running top-KK per query row
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads, 1)
knn_tile_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_l,
                const float* __restrict__ norms, int64_t n, int64_t n_pad, int k_pad, int32_t* __restrict__ cand_idx,
                float* __restrict__ cand_val) {
  extern __shared__ uint8_t smem_raw[];
  // carve: [stages x 64 KB, 1024-aligned] | staged accumulators [128][kAccStride] | norms[2][128] | barriers
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* gen = smem_raw + (base - smem_u32(smem_raw));
  float* s_acc = reinterpret_cast<float*>(gen + kStages * kStageBytes);
  float* s_norm = s_acc + kTileM * kAccStride;
  uint64_t* s_bar = reinterpret_cast<uint64_t*>(s_norm + 2 * kTileN);
  const uint32_t bar0 = smem_u32(s_bar);
  // barriers: full[s] = bar0 + 8 s (TMA bytes landed), empty[s] = bar0 + 16 + 8 s (every consumer warp is done)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int num_kb = k_pad / kBlockK;
  const int num_tiles = (int)(n_pad / kTileN);
  const int row0 = blockIdx.x * kTileM;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(bar0 + 8 * s, 1); mbar_init(bar0 + 16 + 8 * s, kConsumerWarps); }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumerWarps) {
    // ===== TMA producer =====
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0;
      for (int t = 0; t < num_tiles; ++t) {
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(bar0 + 16 + 8 * stage, phase ^ 1);  // slot released by the consumers
          const uint32_t full = bar0 + 8 * stage;
          const uint32_t dst = base + stage * kStageBytes;
          mbar_expect_tx(full, kStageBytes);
          tma_load_2d(dst, &map_h, kb * kBlockK, row0, full);
          tma_load_2d(dst + kOpBytes, &map_l, kb * kBlockK, row0, full);
          tma_load_2d(dst + 2 * kOpBytes, &map_h, kb * kBlockK, t * kTileN, full);
          tma_load_2d(dst + 3 * kOpBytes, &map_l, kb * kBlockK, t * kTileN, full);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumers: warpgroup wg owns query rows row0 + 64 wg .. + 63 =====
  const int wg = warp >> 2;
  const int et = threadIdx.x & 127;            // thread within the warpgroup
  float* acc_s = s_acc + wg * 64 * kAccStride;
  float* sn = s_norm + wg * kTileN;
  // scan: two threads per query row, columns half, half + 2, half + 4, ...
  const int lrow = et >> 1, half = et & 1;
  const int row = row0 + wg * 64 + lrow;
  // accumulator fragment rows / columns of this thread (see wgmma_bf16)
  const int frow = 16 * (warp & 3) + (lane >> 2), fcol = 2 * (lane & 3);

  float bd[kKK];
  int bi[kKK];
#pragma unroll
  for (int q = 0; q < kKK; ++q) { bd[q] = __int_as_float(0x7f800000); bi[q] = -1; }
  float thr = __int_as_float(0x7f800000);
  int worst = 0;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.0f;

  int stage = 0; uint32_t phase = 0;
  for (int t = 0; t < num_tiles; ++t) {
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait(bar0 + 8 * stage, phase);  // operands landed
      const uint32_t sa = base + stage * kStageBytes;
      const uint64_t ah = smem_desc_sw128(sa + wg * 64 * kRowBytes), al = smem_desc_sw128(sa + kOpBytes + wg * 64 * kRowBytes);
      const uint64_t bh = smem_desc_sw128(sa + 2 * kOpBytes), bl = smem_desc_sw128(sa + 3 * kOpBytes);
#pragma unroll
      for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kWgmmaK; ++k) {
        const uint64_t adv = (uint64_t)((k * kWgmmaK * 2) >> 4);  // 32 bytes per K step inside the swizzle atom
        wgmma_bf16(acc, ah + adv, bh + adv, (kb | k) != 0);
        wgmma_bf16(acc, ah + adv, bl + adv, 1u);
        wgmma_bf16(acc, al + adv, bh + adv, 1u);
      }
      wgmma_commit();
      wgmma_wait_all();
#pragma unroll
      for (int i = 0; i < 64; ++i) fence_operand(acc[i]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar0 + 16 + 8 * stage);  // this warp no longer reads the slot
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    // the previous tile's scan of acc_s / sn is finished by every thread of the warpgroup
    named_bar_sync(1 + wg, 128);
#pragma unroll
    for (int j = 0; j < kTileN / 8; ++j) {
      *reinterpret_cast<float2*>(acc_s + frow * kAccStride + 8 * j + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(acc_s + (frow + 8) * kAccStride + 8 * j + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    sn[et] = __ldg(norms + (int64_t)t * kTileN + et);
    named_bar_sync(1 + wg, 128);
    const float* arow = acc_s + lrow * kAccStride;
#pragma unroll 4
    for (int i = 0; i < kTileN / 2; ++i) {
      const int c = 2 * i + half;
      const float dist = fmaf(-2.0f, arow[c], sn[c]);
      if (dist < thr) {
        const int col = t * kTileN + c;
        if (col != row) keep_candidate(bd, bi, dist, col, thr, worst);
      }
    }
  }
  // merge the two half-row lists: the odd-column thread hands its list to the even-column thread
  named_bar_sync(1 + wg, 128);
  float* xd = acc_s + lrow * kAccStride;
  int* xi = reinterpret_cast<int*>(xd + kKK);
  if (half) {
#pragma unroll
    for (int q = 0; q < kKK; ++q) { xd[q] = bd[q]; xi[q] = bi[q]; }
  }
  named_bar_sync(1 + wg, 128);
  if (!half) {
    for (int q = 0; q < kKK; ++q) {
      const float dist = xd[q];
      if (dist < thr) keep_candidate(bd, bi, dist, xi[q], thr, worst);
    }
    if (row < n) {
#pragma unroll
      for (int q = 0; q < kKK; ++q) {
        cand_idx[(int64_t)row * kKK + q] = bi[q];
        cand_val[(int64_t)row * kKK + q] = bd[q];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// re-rank: exact fp32 squared distances of a row's candidates, the k smallest in ascending order
// ---------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
knn_rerank_kernel(const float* __restrict__ X, int64_t n, int d, const int32_t* __restrict__ cand_idx, int k,
                  int32_t* __restrict__ out_idx, float* __restrict__ out_d2) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= n) return;
  const int mine = cand_idx[row * kKK + lane];  // lane q owns candidate q
  float my_d = __int_as_float(0x7f800000);
  const float* xq = X + row * d;
  for (int q = 0; q < kKK; ++q) {
    const int c = __shfl_sync(kFull, mine, q);
    if (c < 0) continue;  // (warp-uniform)
    const float* xc = X + (int64_t)c * d;
    float acc = 0.0f;
    for (int j = lane; j < d; j += 32) { const float t = xq[j] - xc[j]; acc = fmaf(t, t, acc); }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
    if (lane == q) my_d = acc;
  }
  // rank of (my_d, mine) among the 32 candidates: ties broken by index, missing candidates last
  int rank = 0;
  for (int q = 0; q < kKK; ++q) {
    const float od = __shfl_sync(kFull, my_d, q);
    const int oi = __shfl_sync(kFull, mine, q);
    if (q != lane && (od < my_d || (od == my_d && (unsigned)oi < (unsigned)mine))) ++rank;
  }
  if (rank < k) {
    out_idx[row * k + rank] = mine;
    out_d2[row * k + rank] = my_d;
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int make_map(EncodeTiledFn enc, CUtensorMap* map, void* ptr, int64_t n_pad, int k_pad) {
  const cuuint64_t dims[2] = {(cuuint64_t)k_pad, (cuuint64_t)n_pad};
  const cuuint64_t strides[1] = {(cuuint64_t)k_pad * 2};
  const cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)kTileM};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, ptr, dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : MDE_E_INVALID;
}

struct KnnLayout {
  int64_t n_pad; int k_pad;
  size_t off_h, off_l, off_norm, off_ci, off_cv, total;
};

KnnLayout knn_layout(int64_t n, int d) {
  KnnLayout L;
  L.n_pad = (n + kTileN - 1) / kTileN * kTileN;
  L.k_pad = (d + kBlockK - 1) / kBlockK * kBlockK;
  auto up = [](size_t x) { return (x + 1023) / 1024 * 1024; };
  size_t o = 0;
  L.off_h = o; o = up(o + (size_t)L.n_pad * L.k_pad * 2);
  L.off_l = o; o = up(o + (size_t)L.n_pad * L.k_pad * 2);
  L.off_norm = o; o = up(o + (size_t)L.n_pad * 4);
  L.off_ci = o; o = up(o + (size_t)n * kKK * 4);
  L.off_cv = o; o = up(o + (size_t)n * kKK * 4);
  L.total = o;
  return L;
}

}  // namespace

extern "C" {

int mde_knn_max_k(void) { return kMaxK; }

int mde_knn_ws_bytes(int64_t n, int d, size_t* bytes) {
  if (!bytes || n < 2 || d < 1) return MDE_E_INVALID;
  *bytes = knn_layout(n, d).total;
  return 0;
}

int mde_knn(const float* X, int64_t n, int d, int k, int32_t* idx_out, float* d2_out, void* ws, size_t ws_bytes,
            void* stream) {
  if (!X || !idx_out || !d2_out || !ws || n < 2 || d < 1 || k < 1 || k > kMaxK || k > n - 1) return MDE_E_INVALID;
  if (n > (1ll << 31) - kTileN) return MDE_E_UNSUPPORTED;
  const KnnLayout L = knn_layout(n, d);
  if (ws_bytes < L.total || (reinterpret_cast<uintptr_t>(ws) & 1023)) return MDE_E_INVALID;
  cudaStream_t st = (cudaStream_t)stream;
  static EncodeTiledFn enc = nullptr;
  if (!enc) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    MDE_CUDA_TRY(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    if (!fn || qres != cudaDriverEntryPointSuccess) return MDE_E_UNSUPPORTED;
    enc = (EncodeTiledFn)fn;
  }
  uint8_t* w = static_cast<uint8_t*>(ws);
  __nv_bfloat16* Xh = reinterpret_cast<__nv_bfloat16*>(w + L.off_h);
  __nv_bfloat16* Xl = reinterpret_cast<__nv_bfloat16*>(w + L.off_l);
  float* norms = reinterpret_cast<float*>(w + L.off_norm);
  int32_t* ci = reinterpret_cast<int32_t*>(w + L.off_ci);
  float* cv = reinterpret_cast<float*>(w + L.off_cv);
  CUtensorMap mh, ml;
  int rc;
  if ((rc = make_map(enc, &mh, Xh, L.n_pad, L.k_pad))) return rc;
  if ((rc = make_map(enc, &ml, Xl, L.n_pad, L.k_pad))) return rc;
  knn_prep_kernel<<<(unsigned)((L.n_pad + 7) / 8), 256, 0, st>>>(X, n, d, L.n_pad, L.k_pad, Xh, Xl, norms);
  MDE_LAUNCH_CHECK();
  static bool attr_set = false;
  if (!attr_set) {
    MDE_CUDA_TRY(cudaFuncSetAttribute(knn_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
    attr_set = true;
  }
  const unsigned grid = (unsigned)((n + kTileM - 1) / kTileM);
  knn_tile_kernel<<<grid, kThreads, kSmemBytes, st>>>(mh, ml, norms, n, L.n_pad, L.k_pad, ci, cv);
  MDE_LAUNCH_CHECK();
  knn_rerank_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(X, n, d, ci, k, idx_out, d2_out);
  MDE_LAUNCH_CHECK();
  return 0;
}

}  // extern "C"
