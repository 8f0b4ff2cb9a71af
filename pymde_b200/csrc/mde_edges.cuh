// mde_edges.cuh -- the device-resident edge layout shared by mde_edges.cu (layout build, strided / quad / wide
// kernels, per-edge outputs) and mde_tiled.cu (tile-resident kernel).
//
// Layouts (one per shard, chosen at mde_edges_create_ex):
//
//  kind 0  "sorted SoA"     src[p], dst[p], par0[p] (, par1[p]) sorted by (class, src, dst); perm[p].
//                           Any m; the m >= 5 kernels, WeightedQuadratic (par1) and very sparse graphs use it.
//
//  kind 1  "tile records"   m <= 4.  Vertices are cut into dst tiles of R rows (R * m * 8 bytes of X + gradient
//                           fit in one SM's shared memory) and src super-tiles of 2^ss rows (X + gradient of a
//                           super-tile fit in L2).  Edges are grouped into buckets (src super-tile, dst tile),
//                           inside a bucket sorted by (class, src, dst), every bucket padded to whole
//                           "warp-tiles" of 128 edges.  One warp-tile is ONE contiguous 1536-byte record
//                               int32 src[128] | int32 dst[128] | fp32 par0[128]        (pad: dst = -1)
//                           so a warp fetches it with a single cp.async.bulk (TMA) into its shared-memory slot.
//                           perm[nwt * 128] holds the caller position of every slot (-1 for pads).
//
//  kind 3  "SoA + ELL"      m <= 4, n < 2^24, <= 32 neighbour tiles: the kind-0 arrays plus the ELL pull records of
//                           mde_ell.cu (one lane per owner, 12 bytes per edge).
//
//  kind 2  "pull records"   m <= 4.  Same buckets, but every edge is stored as two DIRECTED entries (owner,
//                           neighbour) and a bucket is (owner super-tile, neighbour tile, class); records are
//                           1040 bytes: fp32 w[128] | u16 owner offset[128] | u16 neighbour offset[128] | header
//                           (mde_pull.cu).  No shared-memory atomics, one global red per owner run.
#pragma once
#include "mde_common.cuh"

struct mde_edges {
  int64_t p = 0, n = 0, p_total = 0;
  int kind = 0;
  // ---- kind 0 ----
  int32_t *src = nullptr, *dst = nullptr;
  float *par0 = nullptr, *par1 = nullptr;
  // ---- both ----
  int32_t* perm = nullptr;
  double* loss_partials = nullptr;  // [kMaxLossBlocks]
  mde::FnDev fn;
  int has_par1 = 0;
  int64_t nbytes = 0;
  // kernel switches, resolved once when the layout is created (layouts built with different settings coexist):
  int kvar = 0;              // MDE_B200_KERNEL: 0 default, 1 strided (sorted SoA), 2 precise (no MUFU math)
  int nq = 1;                // MDE_B200_NQ: consecutive quads per thread of the FAST quad kernel (1 or 2)
  int qbps = 4;              // MDE_B200_QUAD_BPS: blocks per SM in the quad kernel's grid cap (1..16)
  int det = 0;               // deterministic mode: gradient contributions accumulate in 64-bit fixed point
  long long* fx = nullptr;   // [n * m_hint] fixed-point accumulator (det only)
  // sorted-SoA layout, m_hint <= 4: every edge is stored again as two directed entries grouped by owner node, and the
  // owner kernel visits each node's entries in this fixed order, keeps the sum in registers and writes the row once
  // (no atomics) -- a gradient that is the same bits from run to run
  uint32_t* inc = nullptr;      // [2 p] (k << 1) | (node is dst), grouped by node: src entries by k, then dst entries by k
  uint2* ent = nullptr;         // [2 p] in the order of inc: (neighbour row | (node is dst) << 31, bits of par0[k])
  int64_t* inc_off = nullptr;   // [n + 1] first entry of node i in inc / ent
  // ---- kind 1 ----
  int m_hint = 0;          // embedding dimension the tile size was chosen for
  int rb = 0;              // log2(R): dst tile rows
  int ss = 0;              // log2(super-tile rows)
  int64_t nwt = 0;         // warp-tiles (128 slots each), padding included
  int32_t* rec = nullptr;  // nwt * 384 words
  int nbkt = 0;            // non-empty buckets
  int32_t* bkt_tile = nullptr;  // [nbkt]     dst tile of bucket b
  int32_t* bkt_wt0 = nullptr;   // [nbkt + 1] first warp-tile of bucket b
  int gred = 0;                 // kind 1: dst contributions as global reds instead of shared-memory CAS
  int ncta = 0;                 // persistent grid of the tile kernel
  int32_t* cta_wt0 = nullptr;   // [ncta + 1] warp-tile range of CTA c
  int32_t* cta_bkt0 = nullptr;  // [ncta]     bucket holding cta_wt0[c]
  // ---- kind 2 (pull records, mde_pull.cu): same bucket / CTA tables, 1040-byte records of DIRECTED entries ----
  int32_t* wt_tile = nullptr;   // [nwt] neighbour tile of every warp-tile (per-edge outputs)
  int epl = 4;                  // entries per lane per warp-tile (a warp-tile holds 32 * epl entries)
  // ---- kind 3 (sorted SoA + ELL pull records, mde_ell.cu): the kind-0 arrays above stay valid ----
  unsigned char* ell_rec = nullptr;   // variable-size records (144 + 192 W bytes)
  uint32_t* ell_off = nullptr;        // [ell_nrec + 1] record offsets, units of 16 bytes
  int32_t *ell_bkt_tile = nullptr, *ell_bkt_wt0 = nullptr;
  int32_t* ell_cta_desc = nullptr;    // [ell_ncta] int4: first record, end record, first bucket, its neighbour tile
  int64_t ell_nrec = 0;
  int ell_ncta = 0;
};

namespace mde {

constexpr int kMaxLossBlocks = kNumSMs * 16;
constexpr int kWtEdges = 128;                 // slots per warp-tile
constexpr int kWtWords = 3 * kWtEdges;        // 32-bit words per record
constexpr int kWtBytes = kWtWords * 4;        // 1536

// tile kernel (mde_tiled.cu)
int tiled_build(mde_edges* e, const int64_t* edges, const float* par0, const mde_fn_t* fn, int embedding_dim,
                cudaStream_t st);
void tiled_free(mde_edges* e);
// MODE 0: fused value + gradient; 1: value only; 2: gradient from caller-ordered per-edge coefficients `gext`
int tiled_launch(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                 int* nblocks_out, const int* flag, cudaStream_t st);
int tiled_edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions,
                       cudaStream_t st);

// pull kernel (mde_pull.cu)
int pull_build(mde_edges* e, const int64_t* edges, const float* par0, const mde_fn_t* fn, int embedding_dim,
               cudaStream_t st);
void pull_free(mde_edges* e);
int pull_launch(int mode, const mde_edges* e, const float* X, int m, float* grad, const float* gext,
                int* nblocks_out, const int* flag, cudaStream_t st);
int pull_edge_outputs(const mde_edges* e, const float* X, int m, float* distances, float* distortions,
                      cudaStream_t st);

// ELL pull kernel (mde_ell.cu): fused value + gradient only; everything else runs on the sorted-SoA kernels
bool ell_supported(int64_t n_items, int embedding_dim);  // shape accepted by the ELL builder (before any allocation)
int ell_build(mde_edges* e, const mde_fn_t* fn, int embedding_dim, cudaStream_t st);
void ell_free(mde_edges* e);
int ell_launch(const mde_edges* e, const float* X, int m, float* grad, int* nblocks_out, const int* flag,
               cudaStream_t st);

}  // namespace mde
