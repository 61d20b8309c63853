// K6+K7 fused: GraphSAGE / EgoSAGE layer forward as ONE persistent, warp-specialised kernel
//
//     out[m, :] = act( [ x_self[m] || agg_j x_nbr[m, j] ] . W^T + b )
//
// One CTA per SM stays resident and walks a static list of row tiles (<= 64 destination rows each)
// that may span SEVERAL segments of the ego graph (e.g. seeds<-hop1 with k=25 and hop1<-hop2 with
// k=10 of a 2-layer GraphSAGE): the tile height of every segment is chosen on the host so that all
// tiles cost about the same number of row fetches and the tile count is a multiple of the SM count.
// Inside the CTA the phases of a tile overlap instead of running back to back:
//
//   gather warps (19)         each warp owns work items (1-4 destination rows x one 512-byte slice): it
//                             translates the item's ids into row pointers (local HBM, a peer GPU's HBM over
//                             NVLink, or the local replica cache) in a private SMEM scratch - the ids of the
//                             NEXT item are prefetched while the current rows are in flight -, pulls the self
//                             row and the k neighbour rows with batches of 16-byte loads, reduces in fp32
//                             registers and writes the bf16 A tile in the wgmma K-major SWIZZLE_128B layout
//                             (and row-major to global for the backward pass); items are dealt round-robin
//                             ACROSS tile boundaries so no warp idles; the A tile is double buffered; rows may be
//                             fp32, bf16 or block-scaled fp8 (dequantised while accumulating)
//   W warp (1)                W image fetched ONCE per CTA by the TMA engine (cp.async.bulk)
//   MMA + epilogue warpgroup (4 warps)  per 32-column slice of the output: wgmma
//                             (M=64, N=32, K=16) over the whole K with the fp32 accumulator in registers,
//                             then bias -> ReLU -> bf16/fp32 store, while the gather warps are already
//                             filling the other A buffer with tile t+1; an mbarrier arrival after the last
//                             slice's MMAs frees the A tile.  For the top layer a second, coalesced phase
//                             (one warp per row, one lane per class) computes the softmax cross-entropy
//                             loss, dlogits and the bias gradient (fused CE)
//
// The rows never round-trip through HBM ("agg(X).W" instead of materialising [B*k, D]).
//
// Math parity: EgoSAGEConv (graphlearn/python/nn/tf/layers/ego_sage_conv.py:71-106):
// agg in {mean,sum,max} over neighbor.reshape(-1,k,d), out = W.[x || agg]; 'gcn' = mean over {x} U nbrs
// then W.  Max is its own instantiation (AGG = kAggMax): the gather warps fold rows with a strict '>' in ascending
// neighbour order and can record, per destination row and column, the first neighbour j holding the maximum (the
// argmax bytes the backward routes the gradient with).  Loss parity: graphlearn/python/nn/tf/loss.py (softmax CE).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cfloat>
#include <cstring>
#include "host_utils.h"
#include "gmma.cuh"
#include "gather_common.cuh"
#include "dropout.cuh"

namespace glb {

constexpr int kTileM = 64;                         // destination rows per tile = wgmma M (two A tiles fit next to the W image)
constexpr int kABufs = 2;
// Role layout: warps [0, 4) = the MMA + epilogue warpgroup, warp 4 = W image loader, warps [5, 24) gather.  The register
// file is split evenly over the CTA's threads, so the layout trades gather warps against row loads in flight per lane:
// 768 threads get 80 registers each, enough for ptxas to issue a whole batch of U loads back to back.
constexpr int kEpiWarps = 4;
constexpr int kWWarp = kEpiWarps;
constexpr int kGatherWarp0 = kEpiWarps + 1;
constexpr int kGatherWarps = 19;
constexpr int kThreads = (kEpiWarps + 1 + kGatherWarps) * 32;
constexpr int kMaxSegs = 4;
constexpr int kScrCap = 64;                        // row pointers per gather warp (private scratch): rows_per_item * (k + 1) <= 64
constexpr size_t kSmemLimit = 232448;

enum SageMode : int { kConcatMean = 0, kConcatSum = 1, kGcnMean = 2, kConcatMax = 3 };
// aggregation of an instantiation: kAggSum serves mean, sum and (sampled mode) gcn, whose scales are runtime factors;
// kAggMax the max; kAggGcn the gcn mean of the CSR mode, which also loads the self row.  kAggSplitK, or-ed into the
// aggregation, marks the instantiations of the split-K launches (a layer whose padded K does not fit one CTA's shared
// memory runs as a self half and a neighbour half, see sage_fused_multi): only they read the split-K fields of SageParams.
enum SageAgg : int { kAggSum = 0, kAggMax = 1, kAggGcn = 2, kAggSplitK = 4 };

struct SageSeg {
  const int64_t* self_vids;   // [M] or null (identity: self_base + m)
  const int64_t* nbr_vids;    // [M, k] or null (identity: nbr_base + m*k + j)
  int64_t self_base, nbr_base;
  char* out;                  // [M, n_out] rows of this segment
  __nv_bfloat16* a_save;      // [M, K_total] or null
  int M, k;
  int R;                      // destination rows per tile (<= 64, multiple of 8)
  int tile0;                  // index of the segment's first tile
};

struct SageParams {
  TableView tself;
  TableView tnbr;
  SageSeg seg[kMaxSegs];
  int nseg, total_tiles;
  const void* w_img;          // bf16 image, (K_total/64) blocks of [N x 64] SW128
  const float* bias;          // [bias_len] or null
  int bias_len;
  int64_t out_stride;         // elements
  int kp_self, kp_nbr;        // padded K of each half, in {0,64,128,256,512}
  int mode;
  int N;                      // padded output width: multiple of 16, <= 256
  int n_out;                  // real output width
  int relu;
  int out_bf16;
  const char* zero_row;       // >= 2 KB of zeros: target of the loads of masked lanes / missing rows
  int wshift_self, wshift_nbr; // log2(world) of each table when it is a power of two, else -1
  // fused softmax cross-entropy (top layer): active when ce_labels != nullptr
  const int64_t* ce_labels;   // label table
  const int64_t* ce_seeds;    // [M] vids (label = ce_labels[seed / ce_world]) or null (label = ce_labels[m])
  int ce_world;
  float* ce_loss;             // accumulated mean loss
  __nv_bfloat16* ce_dlogits;  // [M, ce_dl_stride], columns >= n_out are written as zero
  int ce_dl_stride;
  float* ce_dbias;            // [n_out] accumulated, or null
  float ce_inv_b;
  // several weight images in one launch (an N-split layer): CTA b uses image b % n_imgs, walks the tiles
  // b / n_imgs + j * (gridDim.x / n_imgs) and writes output columns [img * N, img * N + n_out)
  int n_imgs;
  long long* dbg;             // optional [grid][64] clock64 trace (tools/persist_timeline.py), lane 0 of one warp per role
  // CSR neighbour mode (sage_persist_kernel<U, DT, true>, one segment): the neighbours of destination row m are the vids
  // csr_indices[csr_indptr[m] .. csr_indptr[m + 1]); rows with hub_map[m] = h >= 0 instead sum the fp32 partial rows
  // hub_part[hub_cptr[h] .. hub_cptr[h + 1]) of sage_hub_partial_kernel (row stride hub_stride = kp_nbr floats)
  const int64_t* csr_indptr;
  const int64_t* csr_indices;
  const int* hub_map;
  const int* hub_cptr;
  const float* hub_part;
  int hub_stride;
  // max launches: argmax output of segment s (or null), uint8 [M_s, amax_ld], column c = the first j in [0, k) whose
  // neighbour row holds the maximum of column c (kept after the fields above so that their offsets do not move)
  uint8_t* amax[kMaxSegs];
  int amax_ld;
  // inverted dropout of a hidden layer's output (sampled mode), active when drop_state != nullptr: after bias and ReLU,
  // element (row, col) of the layer's output buffer is kept and scaled by drop_scale = 1 / (1 - p) when its 16 mask bits
  // (dropout_bits) are >= drop_thr = round(p * 65536), and zeroed otherwise.  row = drop_row0[s] + m, col = img * N + n.
  const unsigned long long* drop_state;   // {seed, step counter}, 16-byte aligned
  float drop_scale;
  uint32_t drop_thr;
  uint32_t drop_layer;
  int drop_row0[kMaxSegs];
  // split-K launches only (AGG | kAggSplitK).  The layer's images hold both halves ((2 kp / 64) k-blocks each); w_img
  // points at the first k-block of this launch's half in image 0 and w_img_stride (bytes) steps from image to image.
  // a_save rows are the layer's full [self || agg] rows, a_ld elements apart.  The neighbour half adds part[s] (fp32, the
  // self half's output, row stride part_ld, columns as the output's) to its accumulators before bias, ReLU and dropout.
  long long w_img_stride;
  int a_ld;
  const float* part[kMaxSegs];
  int part_ld;
};

// max aggregation: fold one neighbour chunk into the running column maxima
template <int DT, int VEC>
__device__ __forceinline__ void max_into(const Chunk<DT>& c, float (&a)[VEC]) {
  float x[VEC];
  c.get(x);
#pragma unroll
  for (int i = 0; i < VEC; ++i) a[i] = fmaxf(a[i], x[i]);
}

// ... and record the neighbour index j of each new maximum: one byte per column, four to a register.  A strict '>'
// over ascending j keeps the FIRST maximal neighbour (torch.argmax).
template <int DT, int VEC>
__device__ __forceinline__ void max_into(const Chunk<DT>& c, float (&a)[VEC], uint32_t (&ix)[2], uint32_t j) {
  float x[VEC];
  c.get(x);
#pragma unroll
  for (int i = 0; i < VEC; ++i) {
    if (x[i] > a[i]) {
      a[i] = x[i];
      ix[i >> 2] = (ix[i >> 2] & ~(0xFFu << (8 * (i & 3)))) | (j << (8 * (i & 3)));
    }
  }
}

// write VEC consecutive K elements of tile row r starting at K column kcol (multiple of VEC)
template <int VEC>
__device__ __forceinline__ void put_chunk(uint8_t* sA, __nv_bfloat16* a_row, int r, int kcol, const float (&v)[VEC]) {
  const int kb = kcol >> 6;
  const uint32_t off = (uint32_t)kb * (kTileM * 128) + gmma::sw128_offset((uint32_t)r, (uint32_t)(kcol & 63));
  if constexpr (VEC == 4) {
    uint2 u; u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
    *reinterpret_cast<uint2*>(sA + off) = u;
    if (a_row) *reinterpret_cast<uint2*>(a_row + kcol) = u;
  } else {
    uint4 u; u.x = pack_bf16x2(v[0], v[1]); u.y = pack_bf16x2(v[2], v[3]);
    u.z = pack_bf16x2(v[4], v[5]); u.w = pack_bf16x2(v[6], v[7]);
    *reinterpret_cast<uint4*>(sA + off) = u;
    if (a_row) *reinterpret_cast<uint4*>(a_row + kcol) = u;
  }
}

__device__ __forceinline__ int find_seg(const SageParams& p, int t) {
  int s = 0;
#pragma unroll
  for (int i = 1; i < kMaxSegs; ++i)
    if (i < p.nseg && t >= p.seg[i].tile0) s = i;
  return s;
}

#define GLB_DBG(slot) do { if (p.dbg && lane == 0) p.dbg[(size_t)blockIdx.x * 64 + (slot)] = clock64(); } while (0)

// shared-memory control block (after the pointer buffers)
enum : int { kBarW = 0, kBarAFull = 1, kBarAFree = 3, kNumBars = 5 };

// ------------------------------------------------------------------------------------------------
// epilogue of one 32-column slice: wgmma accumulator fragment -> bias/ReLU -> global
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void store_pair(const SageParams& p, const SageSeg& sg, int m, int n, float x0, float x1) {
  if (n >= p.n_out) return;
  const bool two = n + 1 < p.n_out;
  const size_t off = (size_t)m * p.out_stride + n;
  if (p.out_bf16) {
    __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(sg.out) + off;
    if (two && (off & 1) == 0) { *reinterpret_cast<uint32_t*>(o) = pack_bf16x2(x0, x1); return; }
    o[0] = __float2bfloat16(x0);
    if (two) o[1] = __float2bfloat16(x1);
  } else {
    float* o = reinterpret_cast<float*>(sg.out) + off;
    if (two && (off & 1) == 0) { *reinterpret_cast<float2*>(o) = make_float2(x0, x1); return; }
    o[0] = x0;
    if (two) o[1] = x1;
  }
}

// Dropout mask bits of row `row` of a layer's output (dropout_philox in dropout.cuh).
// (Not inlined: inlined, the Philox rounds made ptxas spill 4-40 bytes in the gather roles of several instantiations at
// the 80-register budget; as a call they use the caller's free registers and nothing spills.)
__device__ __noinline__ uint4 dropout_bits(const SageParams& p, uint32_t row, uint32_t col) {
  return dropout_philox(p.drop_state, p.drop_layer, row, col);
}

__device__ __forceinline__ float dropout_apply(const SageParams& p, float x, uint32_t bits16) {
  return bits16 >= p.drop_thr ? x * p.drop_scale : 0.f;
}

// d = the m64n32 accumulator of output columns [n0, n0 + 32) of the tile; bias staged once per CTA in shared memory
// (fp32 [N], zero beyond n_out).  Warp wq of the warpgroup holds rows 16 wq + lane / 4 and 16 wq + lane / 4 + 8.
// row0 = the output buffer row of tile row 0 and c0 = the output column of slice column 0 (dropout only).  DROP = false
// compiles the dropout path out.  The dropout path walks the two rows in a loop that is not unrolled (the same
// register-budget reason as dropout_bits).
template <bool DROP>
__device__ __forceinline__ void sage_epilogue_slice(const SageParams& p, const SageSeg& sg, const float* sBias, const float (&d)[16],
                                                    int m0, int rows, int n0, int wq, int lane, int row0, int c0) {
  const int r0 = wq * 16 + (lane >> 2);
  if (!(DROP && p.drop_state)) {                                   // no dropout: bias -> ReLU -> store
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      const float2 b = *reinterpret_cast<const float2*>(sBias + n);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = r0 + 8 * h;
        float x0 = d[4 * j + 2 * h] + b.x, x1 = d[4 * j + 2 * h + 1] + b.y;
        if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
        if (r < rows) store_pair(p, sg, m0 + r, n, x0, x1);
      }
    }
    return;
  }
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    const int r = r0 + 8 * h;
    const uint4 u = dropout_bits(p, (uint32_t)(row0 + r), (uint32_t)(c0 + n0 + 2 * (lane & 3)));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + 8 * j + 2 * (lane & 3);
      const float2 b = *reinterpret_cast<const float2*>(sBias + n);
      float x0 = (h ? d[4 * j + 2] : d[4 * j]) + b.x, x1 = (h ? d[4 * j + 3] : d[4 * j + 1]) + b.y;
      if (p.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
      const uint32_t w = j == 0 ? u.x : j == 1 ? u.y : j == 2 ? u.z : u.w;
      x0 = dropout_apply(p, x0, w & 0xFFFFu);
      x1 = dropout_apply(p, x1, w >> 16);
      if (r < rows) store_pair(p, sg, m0 + r, n, x0, x1);
    }
  }
}

// phase B (top layer only): softmax cross-entropy of the tile's rows, one warp per row, lanes = classes
// (n_out <= 64: columns lane and lane + 32), reading the logits phase A has just written (L2).
__device__ __forceinline__ void sage_ce_tile(const SageParams& p, const SageSeg& sg, int m0, int rows, int warp, int lane) {
  const float* logits = reinterpret_cast<const float*>(sg.out);
  const int c0 = lane, c1 = lane + 32;
  float db0 = 0.f, db1 = 0.f, lsum = 0.f;
  for (int r = warp; r < rows; r += kEpiWarps) {
    const int m = m0 + r;
    const float* lrow = logits + (size_t)m * p.out_stride;
    const float x0 = c0 < p.n_out ? __ldcg(lrow + c0) : -FLT_MAX;
    const float x1 = c1 < p.n_out ? __ldcg(lrow + c1) : -FLT_MAX;
    long long y = -1;
    if (lane == 0) y = p.ce_seeds ? __ldg(p.ce_labels + __ldg(p.ce_seeds + m) / p.ce_world) : __ldg(p.ce_labels + m);
    y = __shfl_sync(0xffffffffu, y, 0);
    const bool valid = y >= 0 && y < p.n_out;
    float mx = fmaxf(x0, x1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e0 = c0 < p.n_out ? __expf(x0 - mx) : 0.f, e1 = c1 < p.n_out ? __expf(x1 - mx) : 0.f;
    float se = e0 + e1;
    float xy = (c0 == (int)y ? x0 : 0.f) + (c1 == (int)y ? x1 : 0.f);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { se += __shfl_xor_sync(0xffffffffu, se, o); xy += __shfl_xor_sync(0xffffffffu, xy, o); }
    const float inv = 1.f / se;
    const float g0 = (valid && c0 < p.n_out) ? (e0 * inv - (c0 == (int)y ? 1.f : 0.f)) * p.ce_inv_b : 0.f;
    const float g1 = (valid && c1 < p.n_out) ? (e1 * inv - (c1 == (int)y ? 1.f : 0.f)) * p.ce_inv_b : 0.f;
    __nv_bfloat16* drow = p.ce_dlogits + (size_t)m * p.ce_dl_stride;
    if (c0 < p.ce_dl_stride) drow[c0] = __float2bfloat16(g0);
    if (c1 < p.ce_dl_stride) drow[c1] = __float2bfloat16(g1);
    db0 += g0; db1 += g1;
    if (valid) lsum += (mx + __logf(se) - xy) * p.ce_inv_b;
  }
  if (p.ce_dbias) {
    if (c0 < p.n_out && db0 != 0.f) atomicAdd(p.ce_dbias + c0, db0);
    if (c1 < p.n_out && db1 != 0.f) atomicAdd(p.ce_dbias + c1, db1);
  }
  if (lane == 0 && lsum != 0.f) atomicAdd(p.ce_loss, lsum);
}

// ------------------------------------------------------------------------------------------------
// gather-warp helpers
// ------------------------------------------------------------------------------------------------
struct TileCtx {       // kept small on purpose: the gather loop holds two of these next to its row loads
  int s;               // segment index
  int m0, rows;
};

struct GatherGeom {
  int rpi, n_slices, lshift, sub, lig;
  int tile_first, tile_stride;     // this CTA's tiles: tile_first + it * tile_stride
};

// position (it, item) -> first tile at or after `it` in which this warp still has an item; false past the last tile
__device__ __forceinline__ bool seek_item(const SageParams& p, const GatherGeom& gg, int& it, int& item, TileCtx& c) {
  for (;;) {
    const int t = gg.tile_first + it * gg.tile_stride;
    if (t >= p.total_tiles) return false;
    const int s = find_seg(p, t);
    const int m0 = (t - p.seg[s].tile0) * p.seg[s].R;
    const int rows = min(p.seg[s].R, p.seg[s].M - m0);
    const int n_items = ((rows + gg.rpi - 1) >> (5 - gg.lshift)) * gg.n_slices;     // rpi == 32 >> lshift
    if (item < n_items) { c.s = s; c.m0 = m0; c.rows = rows; return true; }
    item -= n_items;
    ++it;
  }
}

// An item holds rpi * (k + 1) ids, flat index f = sub_row * (k + 1) + j (j == k: the self id); a lane owns f = lane and
// f = lane + 32.  The (sub_row, j) split of those two slots only depends on the segment's k: it is cached in
// one byte per slot, (sub_row << 6) | j (0xFF: slot unused; rpi <= 4 and k < 64), both slots packed into one register
// and recomputed when the warp crosses into another segment, so the steady-state loop has no integer division.
__device__ __forceinline__ uint32_t decompose_slots(const GatherGeom& gg, int k, int lane) {
  const int k1 = k + 1;
  const int n_ids = gg.rpi * k1;
  uint32_t dec = 0;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int f = lane + 32 * u;
    const int sr = f / k1;
    dec |= (f < n_ids ? (uint32_t)((sr << 6) | (f - sr * k1)) : 0xFFu) << (8 * u);
  }
  return dec;
}

__device__ __forceinline__ void load_item_ids(const SageParams& p, const GatherGeom& gg, const TileCtx& c, int item, bool need_self,
                                              uint32_t dec, int64_t (&ids)[2]) {
  const SageSeg& sg = p.seg[c.s];
  const int rg = gg.n_slices == 1 ? item : item / gg.n_slices;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    ids[u] = -1;
    const int d = (int)((dec >> (8 * u)) & 0xFFu);
    if (d != 0xFF) {
      const int j = d & 63;
      const int r = rg * gg.rpi + (d >> 6);
      if (r < c.rows) {
        const int64_t m = c.m0 + r;
        if (j < sg.k) ids[u] = sg.nbr_vids ? __ldg(sg.nbr_vids + m * sg.k + j) : sg.nbr_base + m * sg.k + j;
        else if (need_self) ids[u] = sg.self_vids ? __ldg(sg.self_vids + m) : sg.self_base + m;
      }
    }
  }
}

__device__ __forceinline__ void write_item_ptrs(const SageParams& p, const TileCtx& c, const int64_t (&ids)[2], uint32_t dec,
                                                int lane, const char** scr, uint32_t self_row_bytes, uint32_t nbr_row_bytes) {
  const int k = p.seg[c.s].k;
#pragma unroll
  for (int u = 0; u < 2; ++u) {
    const int d = (int)((dec >> (8 * u)) & 0xFFu);
    if (d != 0xFF) {
      scr[lane + 32 * u] = (d & 63) < k ? vid_ptr(p.tnbr, ids[u], p.wshift_nbr, nbr_row_bytes, p.zero_row)
                                             : vid_ptr(p.tself, ids[u], p.wshift_self, self_row_bytes, p.zero_row);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// CSR neighbour mode (layer-wise full-neighbourhood inference): the neighbours of destination row m are the CSR row
// csr_indices[csr_indptr[m] .. csr_indptr[m + 1]) of any length.  An item is ONE destination row x one 512-byte slice:
// the warp's 32 / lpr lane groups split the row's neighbours (group g takes every ngrp-th one) and are summed with
// shuffles at the end, so a warp's time follows the degree of its own row, not the largest of several packed rows.  The
// adjacency is walked in rounds of kScrCap ids: ids -> row pointers (vid_ptr) in the warp's scratch -> U-batched row
// loads.  The id range of the NEXT item is prefetched at the top of an item and its first round of ids right after
// the current row loads.  Hub rows (hub_map >= 0) sum the fp32 partial rows of their adjacency chunks instead.
// AGG = kAggMax takes the column max (lane groups combined with shuffles, 0 for degree 0; hub rows the max of their
// chunks' partial maxima); kAggGcn loads the self row as well and writes (x_self + sum) / (deg + 1).
// ------------------------------------------------------------------------------------------------
template <int U, int DT, int AGG>
__device__ __forceinline__ void sage_csr_gather(const SageParams& p, uint8_t* sA, uint32_t a_buf_bytes, uint64_t* bars,
                                                const char** scr, int tile_first, int tile_stride, int gw, int lane) {
  constexpr int VEC = Chunk<DT>::kVec;
  constexpr uint32_t kEsz = DT == 0 ? 4u : DT == 1 ? 2u : 1u;
  const SageSeg& sg = p.seg[0];
  const int kp = p.kp_nbr > 0 ? p.kp_nbr : p.kp_self;
  const int d_self = p.tself.dim, d_nbr = p.tnbr.dim;
  const int lanes_row = kp / VEC;
  const int lpr = lanes_row < 32 ? lanes_row : 32;
  const int ngrp = 32 / lpr;                            // lane groups sharing the destination row
  const int grp = lane / lpr;
  GatherGeom gg;                                        // one destination row per item
  gg.lshift = 5; gg.rpi = 1; gg.sub = 0;
  gg.n_slices = lanes_row > 32 ? lanes_row >> 5 : 1;
  gg.lig = lane & (lpr - 1);
  gg.tile_first = tile_first; gg.tile_stride = tile_stride;
  constexpr bool kMax = AGG == kAggMax, kGcn = AGG == kAggGcn;
  const bool has_self = p.kp_self > 0, has_nbr = p.kp_nbr > 0;
  const bool need_self = has_self || kGcn;              // gcn: the self row joins the mean (kp_self = 0)
  const uint32_t nbr_row_bytes = (uint32_t)p.tnbr.stride * kEsz, self_row_bytes = (uint32_t)p.tself.stride * kEsz;
  const int soff_self = fp8_scale_offset(d_self), soff_nbr = fp8_scale_offset(d_nbr);
  const int n_tiles_cta = (p.total_tiles - tile_first + tile_stride - 1) / tile_stride;

  int arrived = 0;                                      // as in the sampled gather role
  auto arrive_upto = [&](int upto) {
    while (arrived < upto) {
      gmma::mbar_wait(bars + kBarAFree + (arrived & 1), (uint32_t)(((arrived >> 1) & 1) ^ 1));
      if (lane == 0) gmma::mbar_arrive(bars + kBarAFull + (arrived & 1));
      ++arrived;
    }
  };
  auto fetch_ids = [&](int64_t e0, int64_t e1, int64_t (&v)[2]) {
#pragma unroll
    for (int u = 0; u < 2; ++u) v[u] = e0 + lane + 32 * u < e1 ? __ldg(p.csr_indices + e0 + lane + 32 * u) : -1;
  };

  int it = 0, item = gw;
  TileCtx cur;
  bool valid = seek_item(p, gg, it, item, cur);
  int64_t e_beg = 0, e_end = 0;
  int hub = -1;
  int64_t ids[2] = {-1, -1};                            // first round of ids of the current item
  if (valid) {
    const int m = cur.m0 + (gg.n_slices == 1 ? item : item / gg.n_slices);
    e_beg = __ldg(p.csr_indptr + m); e_end = __ldg(p.csr_indptr + m + 1);
    hub = p.hub_map ? __ldg(p.hub_map + m) : -1;
    if (has_nbr && hub < 0) fetch_ids(e_beg, e_end, ids);
  }
  while (valid) {
    int nit = it, nitem = item + kGatherWarps;
    TileCtx nxt;
    const bool nvalid = seek_item(p, gg, nit, nitem, nxt);
    int64_t nb = 0, ne = 0;
    int nhub = -1;
    if (nvalid) {
      const int nm = nxt.m0 + (gg.n_slices == 1 ? nitem : nitem / gg.n_slices);
      nb = __ldg(p.csr_indptr + nm); ne = __ldg(p.csr_indptr + nm + 1);
      nhub = p.hub_map ? __ldg(p.hub_map + nm) : -1;
    }
    const int rg = gg.n_slices == 1 ? item : item / gg.n_slices;      // row of the tile
    const int sl = gg.n_slices == 1 ? 0 : item - rg * gg.n_slices;
    const int m = cur.m0 + rg;
    const int chunk = gg.lig + 32 * sl;
    const int f0 = chunk * VEC;
    float acc[VEC], sv[VEC];
#pragma unroll
    for (int i = 0; i < VEC; ++i) { acc[i] = kMax ? -INFINITY : 0.f; sv[i] = 0.f; }
    const bool self_ld = need_self && grp == 0 && f0 < d_self;
    Chunk<DT> sraw;
    if (self_ld)
      load_chunk<DT>(sraw, vid_ptr(p.tself, sg.self_vids ? __ldg(sg.self_vids + m) : sg.self_base + m, p.wshift_self,
                                   self_row_bytes, p.zero_row), chunk, soff_self);
    if (has_nbr && hub >= 0) {
      if (f0 < d_nbr) {
        const int c1 = __ldg(p.hub_cptr + hub + 1);
        for (int c = __ldg(p.hub_cptr + hub) + grp; c < c1; c += ngrp) {
          const float4* src = reinterpret_cast<const float4*>(p.hub_part + (size_t)c * p.hub_stride + f0);
#pragma unroll
          for (int q = 0; q < VEC / 4; ++q) {
            const float4 v = __ldcg(src + q);
            if constexpr (kMax) {
              acc[4 * q] = fmaxf(acc[4 * q], v.x); acc[4 * q + 1] = fmaxf(acc[4 * q + 1], v.y);
              acc[4 * q + 2] = fmaxf(acc[4 * q + 2], v.z); acc[4 * q + 3] = fmaxf(acc[4 * q + 3], v.w);
            } else {
              acc[4 * q] += v.x; acc[4 * q + 1] += v.y; acc[4 * q + 2] += v.z; acc[4 * q + 3] += v.w;
            }
          }
        }
      }
    } else if (has_nbr) {
      for (int64_t e0 = e_beg; e0 < e_end; e0 += kScrCap) {
        if (e0 != e_beg) fetch_ids(e0, e_end, ids);
        const int n = (int)(e_end - e0 < kScrCap ? e_end - e0 : kScrCap);
        __syncwarp();                                   // every lane is done reading the previous round's pointers
#pragma unroll
        for (int u = 0; u < 2; ++u)
          if (lane + 32 * u < n) scr[lane + 32 * u] = vid_ptr(p.tnbr, ids[u], p.wshift_nbr, nbr_row_bytes, p.zero_row);
        __syncwarp();
        if (f0 < d_nbr) {
          int j = grp;
          for (; j + (U - 1) * ngrp < n; j += U * ngrp) {
            Chunk<DT> raw[U];
#pragma unroll
            for (int u = 0; u < U; ++u) load_chunk<DT>(raw[u], scr[j + u * ngrp], chunk, soff_nbr);
#pragma unroll
            for (int u = 0; u < U; ++u) {
              if constexpr (kMax) max_into<DT>(raw[u], acc);
              else raw[u].add_to(acc);
            }
          }
          if (j < n) {
            Chunk<DT> raw[U];
#pragma unroll
            for (int u = 0; u < U; ++u) load_chunk<DT>(raw[u], scr[j + u * ngrp < n ? j + u * ngrp : j], chunk, soff_nbr);
#pragma unroll
            for (int u = 0; u < U; ++u) {
              if (j + u * ngrp < n) {
                if constexpr (kMax) max_into<DT>(raw[u], acc);
                else raw[u].add_to(acc);
              }
            }
          }
        }
      }
    }
    if (nvalid && has_nbr && nhub < 0) fetch_ids(nb, ne, ids);
#pragma unroll
    for (int o = lpr; o < 32; o <<= 1)                  // combine the lane groups' shares of the row
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        const float v = __shfl_xor_sync(0xffffffffu, acc[i], o);
        acc[i] = kMax ? fmaxf(acc[i], v) : acc[i] + v;
      }
    if constexpr (kMax) {
      if (e_end == e_beg)                               // degree 0: zero aggregate
#pragma unroll
        for (int i = 0; i < VEC; ++i) acc[i] = 0.f;
    }
    if (self_ld) sraw.add_to(sv);
    if (f0 + VEC > d_self || f0 + VEC > d_nbr) {
#pragma unroll
      for (int i = 0; i < VEC; ++i) {
        if (f0 + i >= d_self) sv[i] = 0.f;
        if (f0 + i >= d_nbr) acc[i] = 0.f;
      }
    }
    arrive_upto(it);
    gmma::mbar_wait(bars + kBarAFree + (it & 1), (uint32_t)(((it >> 1) & 1) ^ 1));
    uint8_t* sAt = sA + (size_t)(it & 1) * a_buf_bytes;
    if (grp == 0) {
      if (has_self) put_chunk<VEC>(sAt, nullptr, rg, f0, sv);
      if (has_nbr) {
        const int64_t deg = e_end - e_beg;              // degree 0: zero aggregate
        if constexpr (kGcn) {
          const float scale = 1.f / (float)(deg + 1);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = (acc[i] + sv[i]) * scale;
        } else {
          const float scale = p.mode == kConcatMean ? (deg > 0 ? 1.f / (float)deg : 0.f) : 1.f;
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] *= scale;
        }
        put_chunk<VEC>(sAt, nullptr, rg, p.kp_self + f0, acc);
      }
    }
    if (!nvalid || nit != it) {                         // last item of this warp in tile `it`
      gmma::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) gmma::mbar_arrive(bars + kBarAFull + (it & 1));
      arrived = it + 1;
    }
    it = nit; item = nitem; cur = nxt; valid = nvalid;
    e_beg = nb; e_end = ne; hub = nhub;
  }
  arrive_upto(n_tiles_cta);
}

// Hub pre-pass of the CSR mode.  The host cuts the adjacency of every row above its hub degree into chunks of a few
// hundred edges (static per CSR); one warp per (chunk, 512-byte slice) sums the chunk's neighbour rows in fp32 into
// part[chunk, 0 .. kp).  The layer launch then reads a hub row's few partial rows instead of its neighbours, so a row of
// 50 000 neighbours is spread over hundreds of warps instead of stalling one gather warp - and with it, through the
// double-buffered A tile, its whole CTA.  Fixed chunking and summation order: the result is deterministic.  MAX: the
// chunk's column maxima instead of sums (a chunk is never empty).
template <int U, int DT, bool MAX>
__global__ void __launch_bounds__(256) sage_hub_partial_kernel(const __grid_constant__ TableView t, int wshift, const int64_t* __restrict__ indices,
                                                               const int64_t* __restrict__ chunks, int n_chunks, int kp,
                                                               float* __restrict__ part, const char* zero_row) {
  constexpr int VEC = Chunk<DT>::kVec;
  constexpr uint32_t kEsz = DT == 0 ? 4u : DT == 1 ? 2u : 1u;
  const int lanes_row = kp / VEC;
  const int lpr = lanes_row < 32 ? lanes_row : 32;
  const int ngrp = 32 / lpr;
  const int n_slices = lanes_row > 32 ? lanes_row >> 5 : 1;
  const int lane = threadIdx.x & 31;
  const int w = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  if (w >= n_chunks * n_slices) return;                // whole warps
  const int c = w / n_slices, sl = w - c * n_slices;
  const int grp = lane / lpr;
  const int chunk = (lane & (lpr - 1)) + 32 * sl;
  const int f0 = chunk * VEC;
  const int64_t e0 = __ldg(chunks + 2 * c);
  const int64_t* ids = indices + e0;
  const int cnt = (int)(__ldg(chunks + 2 * c + 1) - e0);   // <= the host's chunk size
  const uint32_t row_bytes = (uint32_t)t.stride * kEsz;
  const int soff = fp8_scale_offset(t.dim);
  float acc[VEC];
#pragma unroll
  for (int i = 0; i < VEC; ++i) acc[i] = MAX ? -INFINITY : 0.f;
  if (f0 < t.dim) {
    for (int j = grp; j < cnt; j += U * ngrp) {
      const char* ptr[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int ju = j + u * ngrp;
        ptr[u] = ju < cnt ? vid_ptr(t, __ldg(ids + ju), wshift, row_bytes, zero_row) : zero_row;
      }
      Chunk<DT> raw[U];
#pragma unroll
      for (int u = 0; u < U; ++u) load_chunk<DT>(raw[u], ptr[u], chunk, soff);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if constexpr (MAX) {
          if (j + u * ngrp < cnt) max_into<DT>(raw[u], acc);    // (the zero row of a masked load is no candidate)
        } else {
          raw[u].add_to(acc);
        }
      }
    }
  }
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    if (o < lpr) continue;                              // (warp-uniform)
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      const float v = __shfl_xor_sync(0xffffffffu, acc[i], o);
      acc[i] = MAX ? fmaxf(acc[i], v) : acc[i] + v;
    }
  }
  if (grp == 0) {
    float4* dst = reinterpret_cast<float4*>(part + (size_t)c * kp + f0);
#pragma unroll
    for (int q = 0; q < VEC / 4; ++q)
      dst[q] = make_float4(f0 + 4 * q < t.dim ? acc[4 * q] : 0.f, f0 + 4 * q + 1 < t.dim ? acc[4 * q + 1] : 0.f,
                           f0 + 4 * q + 2 < t.dim ? acc[4 * q + 2] : 0.f, f0 + 4 * q + 3 < t.dim ? acc[4 * q + 3] : 0.f);
  }
}

// U  = neighbour row loads kept in flight per lane (one batch)
// DT = storage dtype of the self AND neighbour tables (0 fp32, 1 bf16)
// CSR = neighbour source: fixed-k id lists of the segments (false) or CSR rows of any length (true, sage_csr_gather)
// AGG = SageAgg of the neighbour reduction
//
// Gather decomposition: a row needs LPR = kp / VEC lanes (16-byte chunk per lane); when LPR < 32 a
// warp processes 32/LPR rows side by side (sub-warp groups), when LPR > 32 the row is cut into
// 32-lane slices.  Per item a lane group issues ALL self + neighbour chunk loads of a batch
// unconditionally (masked lanes read a zero row), reduces in fp32 and writes bf16 into the SW128
// A tile.
// DROP: the launch applies dropout (sampled mode only).  A template parameter rather than only the runtime field: with
// the dropout path compiled into every instantiation (and the step counter advanced at p = 0 too) the headline step
// measured 1.6 % slower at p = 0.
// AGG | kAggSplitK: one half of a split-K layer (image stride, a_save row stride and, for the neighbour half, the self
// half's fp32 partial added before the epilogue).
template <int U, int DT, bool CSR, int AGG, bool DROP>
__global__ void __launch_bounds__(kThreads, 1) sage_persist_kernel(const __grid_constant__ SageParams p) {
  constexpr int kAgg = AGG & ~kAggSplitK;
  constexpr bool kSplit = (AGG & kAggSplitK) != 0;
  if (p.dbg && threadIdx.x == 0) {
    unsigned long long gt; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    p.dbg[(size_t)blockIdx.x * 64 + 60] = (long long)gt;
    p.dbg[(size_t)blockIdx.x * 64 + 61] = clock64();
  }
  // keep every pointer derived from the __shared__ symbol by plain integer offsets so that the
  // compiler emits LDS/STS (a uintptr_t round trip would demote them to generic LD/ST)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (gmma::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int k_total = p.kp_self + p.kp_nbr;
  const int nkb = k_total >> 6;
  uint8_t* sA = smem;
  const uint32_t a_buf_bytes = (uint32_t)nkb * (kTileM * 128);
  uint8_t* sW = sA + (size_t)kABufs * a_buf_bytes;
  const uint32_t w_kb_bytes = (uint32_t)p.N * 128u;
  const char** sScr = reinterpret_cast<const char**>(sW + (size_t)nkb * w_kb_bytes);   // [kGatherWarps][kScrCap]
  float* sBias = reinterpret_cast<float*>(sScr + kGatherWarps * kScrCap);              // [256]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sBias + 256);

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;

  if (tid == 0) {
    gmma::mbar_init(bars + kBarW, 1);
    for (int i = 0; i < 2; ++i) {
      gmma::mbar_init(bars + kBarAFull + i, kGatherWarps);
      gmma::mbar_init(bars + kBarAFree + i, kEpiWarps);
    }
    gmma::fence_barrier_init();
  }
  const int img = (int)blockIdx.x % p.n_imgs;
  // (multi-image launches: image `img` owns the output columns [img * N, img * N + N) and the matching bias slice)
  if (tid < 256) sBias[tid] = (p.bias && tid < p.n_out && img * p.N + tid < p.bias_len) ? __ldg(p.bias + img * p.N + tid) : 0.f;
  __syncthreads();
  const int tile_first = (int)blockIdx.x / p.n_imgs, tile_stride = (int)gridDim.x / p.n_imgs;
  if (warp == 0) GLB_DBG(0);

  if (warp < kEpiWarps) {
    // =================================================================== MMA + epilogue warpgroup
    gmma::mbar_wait(bars + kBarW, 0);
    const uint32_t w_base = gmma::smem_u32(sW);
    // padded output columns are never read back: slices past n_out are not computed
    const int n_slices = (min(p.N, (p.n_out + 31) & ~31)) >> 5;
    int it = 0;
    for (int t = tile_first; t < p.total_tiles; t += tile_stride, ++it) {
      const int buf = it & 1;
      gmma::mbar_wait(bars + kBarAFull + buf, (uint32_t)((it >> 1) & 1));
      if (warp == 0 && it < 4) GLB_DBG(4 + it * 2);
      const int s = find_seg(p, t);
      SageSeg sg = p.seg[s];
      if (sg.out) sg.out += (size_t)img * p.N * (p.out_bf16 ? 2 : 4);
      const int m0 = (t - sg.tile0) * sg.R;
      const int rows = min(sg.R, sg.M - m0);
      const uint32_t a_base = gmma::smem_u32(sA + (size_t)buf * a_buf_bytes);
      for (int sl = 0; sl < n_slices; ++sl) {
        float d[16];
        gmma::wgmma_fence();
        for (int kb = 0; kb < nkb; ++kb) {
          const uint32_t a_kb = a_base + (uint32_t)kb * (kTileM * 128);
          const uint32_t b_kb = w_base + (uint32_t)kb * w_kb_bytes + (uint32_t)sl * (32 * 128);
#pragma unroll
          for (int k4 = 0; k4 < 4; ++k4)
            gmma::mma_m64n32_bf16<0, 0>(d, gmma::make_desc_sw128(a_kb + k4 * 32), gmma::make_desc_sw128(b_kb + k4 * 32), (kb | k4) ? 1u : 0u);
        }
        gmma::wgmma_commit();
        gmma::wgmma_wait<0>();
        gmma::fence_regs(d);
        if (sl == n_slices - 1) {                         // this warp's last MMA on the A tile has completed
          __syncwarp();
          if (lane == 0) gmma::mbar_arrive(bars + kBarAFree + buf);
        }
        if constexpr (kSplit) {                           // neighbour half: + the self half's x_self . W_self^T
          const float* part = p.part[s];
          if (part != nullptr) {
            const int r0 = (warp & 3) * 16 + (lane >> 2);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              if (r0 + 8 * h >= rows) continue;
              const float* prow = part + (size_t)(m0 + r0 + 8 * h) * p.part_ld + img * p.N + sl * 32 + 2 * (lane & 3);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const float2 v = __ldcg(reinterpret_cast<const float2*>(prow + 8 * j));
                d[4 * j + 2 * h] += v.x;
                d[4 * j + 2 * h + 1] += v.y;
              }
            }
          }
        }
        // (warp < 4 here; the mask tells the compiler so: without it the <6, bf16> instantiation spills at 80 registers)
        if (sg.out) sage_epilogue_slice<DROP>(p, sg, sBias, d, m0, rows, sl * 32, warp & 3, lane, p.drop_row0[s] + m0, img * p.N);
      }
      if (p.ce_labels != nullptr) {
        __threadfence_block();
        asm volatile("bar.sync 1, %0;" ::"r"(kEpiWarps * 32) : "memory");     // logits of the tile are written
        sage_ce_tile(p, sg, m0, rows, warp, lane);
      }
      if (warp == 0 && it < 4) GLB_DBG(5 + it * 2);
    }
  } else if (warp == kWWarp) {
    // =================================================================== W image via TMA
    if (lane == 0) {
      gmma::mbar_arrive_expect_tx(bars + kBarW, (uint32_t)nkb * w_kb_bytes);
      const uint8_t* src = reinterpret_cast<const uint8_t*>(p.w_img) +
                           (kSplit ? (size_t)img * (size_t)p.w_img_stride : (size_t)img * nkb * w_kb_bytes);
      for (int kb = 0; kb < nkb; ++kb)
        gmma::bulk_g2s(sW + (size_t)kb * w_kb_bytes, src + (size_t)kb * w_kb_bytes, w_kb_bytes, bars + kBarW);
    }
    __syncwarp();
    gmma::mbar_wait(bars + kBarW, 0);
    GLB_DBG(1);
  } else if constexpr (CSR) {
    sage_csr_gather<U, DT, kAgg>(p, sA, a_buf_bytes, bars, sScr + (warp - kGatherWarp0) * kScrCap, tile_first, tile_stride,
                                 warp - kGatherWarp0, lane);
  } else {
    // =================================================================== gather warps
    constexpr int VEC = Chunk<DT>::kVec;
    constexpr bool kMax = kAgg == kAggMax;
    const int gw = warp - kGatherWarp0;
    const int kp = p.kp_nbr > 0 ? p.kp_nbr : p.kp_self;
    const int d_self = p.tself.dim, d_nbr = p.tnbr.dim;
    const int lanes_row = kp / VEC;                       // 16-byte chunks per (half) row: 8..128
    const int lpr = lanes_row < 32 ? lanes_row : 32;      // lanes per row inside a warp
    GatherGeom gg;
    gg.lshift = 31 - __clz(lpr);                          // log2(lpr)
    gg.rpi = 32 >> gg.lshift;                             // rows per item
    gg.n_slices = lanes_row > 32 ? lanes_row >> 5 : 1;
    gg.sub = lane >> gg.lshift;                           // which row of the item this lane works on
    gg.lig = lane & (lpr - 1);                            // lane index inside its row group
    gg.tile_first = tile_first; gg.tile_stride = tile_stride;
    const bool has_self = p.kp_self > 0;
    const bool has_nbr = p.kp_nbr > 0;
    const bool need_self = has_self || p.mode == kGcnMean;
    constexpr uint32_t kEsz = DT == 0 ? 4u : DT == 1 ? 2u : 1u;
    const uint32_t nbr_row_bytes = (uint32_t)p.tnbr.stride * kEsz;
    const uint32_t self_row_bytes = (uint32_t)p.tself.stride * kEsz;
    const int soff_self = fp8_scale_offset(d_self), soff_nbr = fp8_scale_offset(d_nbr);     // fp8 rows: where the block scales start
    const char** scr = sScr + gw * kScrCap;
    const int n_tiles_cta = (p.total_tiles - tile_first + tile_stride - 1) / tile_stride;

    int arrived = 0;                                      // tiles this warp has already arrived for on a_full
    // arrive for every tile < upto (tiles in which this warp has no item left); an arrival for tile j (A buffer
    // j & 1) is only legal once the MMA of tile j-2 has been committed, otherwise it would be counted in that
    // tile's phase (a fresh barrier passes the parity-1 wait, so tiles 0 and 1 need no special case)
    auto arrive_upto = [&](int upto) {
      while (arrived < upto) {
        gmma::mbar_wait(bars + kBarAFree + (arrived & 1), (uint32_t)(((arrived >> 1) & 1) ^ 1));
        if (lane == 0) gmma::mbar_arrive(bars + kBarAFull + (arrived & 1));
        ++arrived;
      }
    };

    int it = 0, item = gw;
    TileCtx cur;
    bool valid = seek_item(p, gg, it, item, cur);
    uint32_t dec = 0xFFFFu;                               // id-slot split of the segment `dec_seg`
    int dec_seg = -1;
    if (valid) {
      int64_t ids[2];
      dec_seg = cur.s;
      dec = decompose_slots(gg, p.seg[cur.s].k, lane);
      load_item_ids(p, gg, cur, item, need_self, dec, ids);
      write_item_ptrs(p, cur, ids, dec, lane, scr, self_row_bytes, nbr_row_bytes);
      __syncwarp();
    }
    if (gw == 0) GLB_DBG(28);
    while (valid) {
      // ---- prefetch the ids of this warp's NEXT item (their latency hides behind the row loads below)
      int nit = it, nitem = item + kGatherWarps;
      TileCtx nxt;
      const bool nvalid = seek_item(p, gg, nit, nitem, nxt);
      int64_t nids[2];
      if (nvalid) {
        // (the current item's pointers are already staged: `dec` only serves the NEXT item from here on)
        if (nxt.s != dec_seg) { dec = decompose_slots(gg, p.seg[nxt.s].k, lane); dec_seg = nxt.s; }   // rare
        load_item_ids(p, gg, nxt, nitem, need_self, dec, nids);
      }
      // ---- current item
      const SageSeg& sg = p.seg[cur.s];
      const int k = sg.k;
      const int rg = gg.n_slices == 1 ? item : item / gg.n_slices;
      const int sl = gg.n_slices == 1 ? 0 : item - rg * gg.n_slices;
      const int r = rg * gg.rpi + gg.sub;
      const bool row_ok = r < cur.rows;
      const int chunk = gg.lig + 32 * sl;                 // this lane's 16-byte chunk of the row
      const int f0 = chunk * VEC;                         // first feature of the chunk
      float acc[VEC], sv[VEC];
      uint32_t ix[2] = {0u, 0u};                          // (max) argmax bytes of the chunk's columns
#pragma unroll
      for (int i = 0; i < VEC; ++i) { acc[i] = 0.f; sv[i] = 0.f; }
      if (row_ok) {
        // lanes whose chunk lies beyond the real feature width skip the loads altogether (their A
        // columns are the zero K-padding); the others issue self + U neighbour loads back to back
        const char* const* ptrs = scr + gg.sub * (k + 1);
        const bool self_ld = need_self && f0 < d_self;
        Chunk<DT> sraw;
        if (self_ld) load_chunk<DT>(sraw, ptrs[k], chunk, soff_self);
        if (has_nbr && f0 < d_nbr) {
          if constexpr (kMax) {                           // k = 0 keeps the zero aggregate
            if (k > 0)
#pragma unroll
              for (int i = 0; i < VEC; ++i) acc[i] = -INFINITY;
          }
          int j0 = 0;
          for (; j0 + U <= k; j0 += U) {                  // full batches: U unconditional loads, then U adds
            Chunk<DT> raw[U];
#pragma unroll
            for (int u = 0; u < U; ++u) load_chunk<DT>(raw[u], ptrs[j0 + u], chunk, soff_nbr);
#pragma unroll
            for (int u = 0; u < U; ++u) {                 // (max: ascending j, so the first maximal row wins)
              if constexpr (kMax) max_into<DT>(raw[u], acc, ix, (uint32_t)(j0 + u));
              else raw[u].add_to(acc);
            }
          }
          if (j0 < k) {                                   // remainder batch (k % U rows)
            Chunk<DT> raw[U];
#pragma unroll
            for (int u = 0; u < U; ++u) load_chunk<DT>(raw[u], ptrs[j0 + u < k ? j0 + u : k - 1], chunk, soff_nbr);
#pragma unroll
            for (int u = 0; u < U; ++u) {
              if (j0 + u < k) {
                if constexpr (kMax) max_into<DT>(raw[u], acc, ix, (uint32_t)(j0 + u));
                else raw[u].add_to(acc);
              }
            }
          }
        }
        if (self_ld) sraw.add_to(sv);
        if (f0 + VEC > d_self || f0 + VEC > d_nbr) {       // only the chunk that straddles the real width needs masking
#pragma unroll
          for (int i = 0; i < VEC; ++i) {
            if (f0 + i >= d_self) sv[i] = 0.f;
            if (f0 + i >= d_nbr) acc[i] = 0.f;
          }
        }
      }
      // ---- A buffer it & 1 may only be written once the MMA of tile it-2 has consumed it
      arrive_upto(it);
      gmma::mbar_wait(bars + kBarAFree + (it & 1), (uint32_t)(((it >> 1) & 1) ^ 1));
      uint8_t* sAt = sA + (size_t)(it & 1) * a_buf_bytes;
      if (row_ok) {
        const int m = cur.m0 + r;
        __nv_bfloat16* a_row = (sg.a_save && img == 0) ? sg.a_save + (size_t)m * (kSplit ? p.a_ld : k_total) : nullptr;
        if (has_self) put_chunk<VEC>(sAt, a_row, r, f0, sv);
        if (has_nbr) {
          float scale = 1.f;
          if (p.mode == kConcatMean) scale = k > 0 ? 1.f / (float)k : 0.f;
          else if (p.mode == kGcnMean) scale = 1.f / (float)(k + 1);
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[i] = (acc[i] + (p.mode == kGcnMean ? sv[i] : 0.f)) * scale;
          put_chunk<VEC>(sAt, a_row, r, p.kp_self + f0, acc);
        }
        if constexpr (kMax) {
          uint8_t* am = p.amax[cur.s];
          if (am != nullptr && img == 0 && has_nbr && f0 < d_nbr) {
            uint8_t* dst = am + (size_t)m * p.amax_ld + f0;
            if constexpr (VEC == 8) *reinterpret_cast<uint2*>(dst) = make_uint2(ix[0], ix[1]);
            else *reinterpret_cast<uint32_t*>(dst) = ix[0];
          }
        }
      }
      if (!nvalid || nit != it) {                         // last item of this warp in tile `it`
        gmma::fence_proxy_async_smem();                   // generic-proxy st.shared -> visible to wgmma (async proxy)
        __syncwarp();
        if (lane == 0) gmma::mbar_arrive(bars + kBarAFull + (it & 1));
        arrived = it + 1;
        if (gw == 0 && it < 4) GLB_DBG(30 + it * 3);
      }
      __syncwarp();                                       // every lane is done reading the scratch pointers
      if (nvalid) {
        write_item_ptrs(p, nxt, nids, dec, lane, scr, self_row_bytes, nbr_row_bytes);
        __syncwarp();
      }
      it = nit; item = nitem; cur = nxt; valid = nvalid;
    }
    arrive_upto(n_tiles_cta);
  }
  __syncthreads();
  if (warp == 0) GLB_DBG(2);
  if (p.dbg && threadIdx.x == 0) {
    unsigned long long gt; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    p.dbg[(size_t)blockIdx.x * 64 + 62] = (long long)gt;
  }
}

// fp32 row-major padded weight [n_real, k_total] -> (SW128 bf16 image, bf16 row-major copy) in one pass
__global__ void pack_sw128_f32_kernel(const float* __restrict__ w, int n_real, int N, int k_total,
                                      uint8_t* __restrict__ img, __nv_bfloat16* __restrict__ w16) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;   // one 16-byte (8 element) chunk each
  int nkb = k_total >> 6;
  int total = nkb * N * 8;
  if (idx >= total) return;
  int c = idx & 7;
  int n = (idx >> 3) % N;
  int kb = (idx >> 3) / N;
  uint4 val = make_uint4(0, 0, 0, 0);
  if (n < n_real) {
    const float4* src = reinterpret_cast<const float4*>(w + (size_t)n * k_total + kb * 64 + c * 8);
    float4 a = src[0], b = src[1];
    val.x = pack_bf16x2(a.x, a.y); val.y = pack_bf16x2(a.z, a.w);
    val.z = pack_bf16x2(b.x, b.y); val.w = pack_bf16x2(b.z, b.w);
    if (w16) *reinterpret_cast<uint4*>(w16 + (size_t)n * k_total + kb * 64 + c * 8) = val;
  }
  size_t off = (size_t)kb * N * 128 + (size_t)(n >> 3) * 1024 + (size_t)(n & 7) * 128 + (size_t)((c ^ (n & 7)) * 16);
  *reinterpret_cast<uint4*>(img + off) = val;
}

// ---------------------------------------------------------------------------
static int pad_k(int d) {
  if (d <= 0) return 0;
  if (d <= 64) return 64;
  if (d <= 128) return 128;
  if (d <= 256) return 256;
  TORCH_CHECK(d <= 512, "fused SAGE layer supports feature dims up to 512");
  return 512;
}

// dynamic shared memory of the persistent kernel: A tile + W image + per-warp pointer scratch + bias + control + alignment slack
// (ops/sage.py smem_bytes mirrors this term for term)
int64_t sage_smem_bytes(int64_t k_total, int64_t N) {
  return 1024 + kABufs * (k_total / 64) * (kTileM * 128) + (k_total / 64) * N * 128 + kGatherWarps * kScrCap * 8 + 256 * 4 + (kNumBars + 2) * 8;
}

int sm_count() {
  static int n = 0;
  if (n == 0) n = at::cuda::getCurrentDeviceProperties()->multiProcessorCount;
  return n;
}

// returns (image, bf16 row-major copy)
std::vector<at::Tensor> pack_weight_f32(const at::Tensor& w_padded, int64_t N, bool want_rowmajor) {
  TORCH_CHECK(w_padded.is_cuda() && w_padded.scalar_type() == at::kFloat && w_padded.dim() == 2 &&
              w_padded.is_contiguous(), "w_padded must be a contiguous CUDA fp32 [n, k_total] tensor");
  int64_t n_real = w_padded.size(0), k_total = w_padded.size(1);
  TORCH_CHECK(k_total % 64 == 0 && N % 8 == 0 && N >= n_real, "bad padded weight shape");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(w_padded.data_ptr()) & 15) == 0, "weight must be 16 B aligned");
  c10::cuda::CUDAGuard guard(w_padded.device());
  auto o16 = w_padded.options().dtype(at::kBFloat16);
  auto img = at::empty({(k_total / 64) * N * 64}, o16);
  at::Tensor w16;
  if (want_rowmajor) w16 = at::empty({n_real, k_total}, o16);
  int total = (int)((k_total / 64) * N * 8);
  pack_sw128_f32_kernel<<<(total + 255) / 256, 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      w_padded.data_ptr<float>(), (int)n_real, (int)N, (int)k_total, reinterpret_cast<uint8_t*>(img.data_ptr()),
      want_rowmajor ? reinterpret_cast<__nv_bfloat16*>(w16.data_ptr()) : nullptr);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {img, want_rowmajor ? w16 : at::Tensor()};
}

static long long* g_dbg_ptr = nullptr;
void sage_set_debug_trace(const c10::optional<at::Tensor>& t) {
  g_dbg_ptr = (t.has_value() && t->defined()) ? reinterpret_cast<long long*>(t->data_ptr<int64_t>()) : nullptr;
}

static int log2_or_neg(int w) { int s = 0; while ((1 << s) < w) ++s; return (1 << s) == w ? s : -1; }

static const char* zero_row_for(const at::TensorOptions& opts, int dev) {
  static std::vector<at::Tensor> zero_rows(64);
  if (!zero_rows[dev].defined()) zero_rows[dev] = at::zeros({1024}, opts.dtype(at::kFloat));
  return reinterpret_cast<const char*>(zero_rows[dev].data_ptr());
}

// Balanced tiling: every tile should cost about the same number of row fetches ((k + 1) per destination
// row, + 2 for the epilogue / A stores) and the tile count should just fill `waves` tiles per SM.
static void plan_tiles(SageParams& p) {
  const int sms = std::max(1, sm_count() / p.n_imgs);
  int64_t n128 = 0;
  double total_cost = 0.0;
  for (int s = 0; s < p.nseg; ++s) {
    n128 += (p.seg[s].M + kTileM - 1) / kTileM;
    total_cost += (double)p.seg[s].M * (p.seg[s].k + 3);
  }
  const int64_t waves = std::max<int64_t>(1, (n128 + sms - 1) / sms);
  const double target = total_cost / (double)(sms * waves);
  int tiles = 0;
  for (int s = 0; s < p.nseg; ++s) {
    SageSeg& sg = p.seg[s];
    int64_t R = (int64_t)std::ceil(target / (double)(sg.k + 3));
    R = (R + 7) / 8 * 8;
    R = std::min<int64_t>(kTileM, std::max<int64_t>(8, R));
    sg.R = (int)R;
    sg.tile0 = tiles;
    tiles += sg.M > 0 ? (int)((sg.M + R - 1) / R) : 0;
  }
  p.total_tiles = tiles;
}

template <int U, int DT, bool CSR, int AGG, bool DROP = false>
static void launch_one(const SageParams& p, unsigned grid, size_t smem, cudaStream_t stream) {
  static bool attr_done = false;
  if (!attr_done) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(sage_persist_kernel<U, DT, CSR, AGG, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemLimit));
    attr_done = true;
  }
  sage_persist_kernel<U, DT, CSR, AGG, DROP><<<grid, kThreads, smem, stream>>>(p);
}

// row loads in flight per lane of the CSR mode (one instantiation per table dtype)
constexpr int kCsrU = 5;

static void launch_persist(SageParams& p, size_t smem, cudaStream_t stream, bool csr = false, bool split = false) {
  if (p.total_tiles == 0) return;
  const unsigned grid = (unsigned)(p.n_imgs * std::min<int>(std::max(1, sm_count() / p.n_imgs), p.total_tiles));
  int kmax = 1;
  for (int s = 0; s < p.nseg; ++s) kmax = std::max(kmax, p.seg[s].k);
  const int dt = p.tnbr.dtype;
#define LAUNCH_DT3(UU, CC, AA, DD) do { if (dt == 2) launch_one<UU, 2, CC, AA, DD>(p, grid, smem, stream); \
                                        else if (dt == 0) launch_one<UU, 0, CC, AA, DD>(p, grid, smem, stream); \
                                        else launch_one<UU, 1, CC, AA, DD>(p, grid, smem, stream); } while (0)
#define LAUNCH_U(AA, DD) do { if (u == 4) LAUNCH_DT3(4, false, AA, DD); else if (u == 5) LAUNCH_DT3(5, false, AA, DD); \
                              else LAUNCH_DT3(6, false, AA, DD); } while (0)
  const int u = kmax <= 4 ? 4 : (kmax % 5 == 0 || kmax > 12) ? 5 : 6;
  const bool drop = p.drop_state != nullptr;
  constexpr int kSumS = kAggSum | kAggSplitK, kMaxS = kAggMax | kAggSplitK;
  if (split && csr) {
    if (p.mode == kConcatMax) LAUNCH_DT3(kCsrU, true, kMaxS, false);
    else LAUNCH_DT3(kCsrU, true, kSumS, false);
  } else if (split) {
    // (U = 4 or 5 only: at U = 6 the max + dropout instantiations spill at 80 registers next to the partial's loads)
#define LAUNCH_U45(AA, DD) do { if (u == 4) LAUNCH_DT3(4, false, AA, DD); else LAUNCH_DT3(5, false, AA, DD); } while (0)
    if (p.mode == kConcatMax) { if (drop) LAUNCH_U45(kMaxS, true); else LAUNCH_U45(kMaxS, false); }
    else if (drop) LAUNCH_U45(kSumS, true); else LAUNCH_U45(kSumS, false);
#undef LAUNCH_U45
  } else if (csr) {
    if (p.mode == kConcatMax) LAUNCH_DT3(kCsrU, true, kAggMax, false);
    else if (p.mode == kGcnMean) LAUNCH_DT3(kCsrU, true, kAggGcn, false);
    else LAUNCH_DT3(kCsrU, true, kAggSum, false);
  } else if (p.mode == kConcatMax) {
    if (drop) LAUNCH_U(kAggMax, true); else LAUNCH_U(kAggMax, false);
  } else if (drop) LAUNCH_U(kAggSum, true); else LAUNCH_U(kAggSum, false);
#undef LAUNCH_U
#undef LAUNCH_DT3
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// Launch-wide fields and checks shared by both entry points: tables, padded K, weight image, bias, output format.
// split_half: 0 = the whole layer; 1 / 2 = the self / neighbour half of a split-K layer (a mean, sum or max layer
// whose halves are padded alike), whose images hold both halves.  Returns the dynamic shared memory of the launch; `b`
// keeps a contiguous copy of the bias alive.
static size_t init_layer_params(SageParams& p, const at::Tensor& tself_desc, const at::Tensor& tnbr_desc, bool any_nbr, int64_t mode,
                                const at::Tensor& w_img, const c10::optional<at::Tensor>& bias, at::Tensor& b, int64_t N,
                                int64_t n_out, bool relu, bool out_bf16, int64_t n_imgs, int64_t split_half = 0) {
  std::memset(&p, 0, sizeof(p));
  p.tself = table_from_desc(tself_desc);
  p.tnbr = table_from_desc(tnbr_desc);
  p.mode = (int)mode;
  TORCH_CHECK(split_half >= 0 && split_half <= 2, "split_half must be 0 (whole layer), 1 (self half) or 2 (neighbour half)");
  if (split_half != 0)
    TORCH_CHECK(mode != kGcnMean && pad_k(p.tself.dim) == pad_k(p.tnbr.dim),
                "a split-K layer aggregates with mean, sum or max over equally padded self / neighbour inputs");
  p.kp_self = (mode == kGcnMean || split_half == 2) ? 0 : pad_k(p.tself.dim);
  p.kp_nbr = (any_nbr && split_half != 1) ? pad_k(p.tnbr.dim) : 0;
  if (mode == kGcnMean) TORCH_CHECK(p.tself.dim == p.tnbr.dim, "gcn mode needs equal dims");
  const int k_total = p.kp_self + p.kp_nbr;
  TORCH_CHECK(k_total >= 64, "empty layer");
  TORCH_CHECK(N % 32 == 0 && N >= 32 && N <= 256, "padded N must be a multiple of 32 in [32, 256]");
  TORCH_CHECK(n_out <= N && n_out >= 1);
  TORCH_CHECK(n_imgs >= 1 && n_imgs <= 8 && (n_imgs == 1 || n_out == N), "bad image count");
  p.n_imgs = (int)n_imgs;
  const int64_t k_layer = split_half != 0 ? 2 * (int64_t)k_total : k_total;      // K of the layer's images
  TORCH_CHECK(w_img.numel() == n_imgs * k_layer * N, "weight image size mismatch: expected ", n_imgs * k_layer * N, " got ", w_img.numel());
  TORCH_CHECK((reinterpret_cast<uintptr_t>(w_img.data_ptr()) & 15) == 0, "weight image must be 16 B aligned");
  const size_t smem = (size_t)sage_smem_bytes(k_total, N);
  TORCH_CHECK(smem <= kSmemLimit, "tile does not fit in shared memory (", smem, " B); use the unfused path");
  TORCH_CHECK(p.tself.dtype == p.tnbr.dtype, "fused SAGE layer needs self / neighbour tables of the same storage dtype");
  TORCH_CHECK(p.kp_self == 0 || p.kp_nbr == 0 || p.kp_self == p.kp_nbr, "fused SAGE layer needs equally padded self / neighbour dims");
  TORCH_CHECK((p.tself.stride * table_esize(p.tself.dtype)) % 16 == 0 && (p.tnbr.stride * table_esize(p.tnbr.dtype)) % 16 == 0,
              "table rows must be 16-byte aligned (stride multiple of 4 fp32 / 8 bf16 elements)");
  if (bias.has_value() && bias->defined()) {
    b = bias->contiguous();
    TORCH_CHECK(b.is_cuda() && b.scalar_type() == at::kFloat && (n_imgs > 1 || b.numel() >= n_out), "bias must be fp32 [>= n_out]");
    p.bias = b.data_ptr<float>();
    p.bias_len = (int)b.numel();
  }
  p.w_img = w_img.data_ptr();
  if (split_half != 0) {              // image i = (2 kp / 64) k-blocks of [N x 64]: the self half's, then the neighbour half's
    p.w_img_stride = (long long)(k_layer / 64) * N * 128;
    if (split_half == 2) p.w_img = reinterpret_cast<const char*>(w_img.data_ptr()) + (size_t)(k_total / 64) * N * 128;
  }
  p.N = (int)N; p.n_out = (int)n_out; p.relu = relu ? 1 : 0; p.out_bf16 = out_bf16 ? 1 : 0;
  p.wshift_self = log2_or_neg(p.tself.world);
  p.wshift_nbr = log2_or_neg(p.tnbr.world);
  p.zero_row = zero_row_for(w_img.options(), w_img.get_device());
  return smem;
}

// output rows of one segment (an undefined tensor: no output); every segment of a launch shares the row stride
static void set_seg_out(SageParams& p, SageSeg& sg, const at::Tensor& out, int64_t M, int64_t n_out, bool out_bf16) {
  if (!out.defined()) return;
  TORCH_CHECK(out.is_cuda() && out.dim() == 2 && out.size(0) == M && out.size(1) == n_out && out.stride(1) == 1,
              "outs[i] must be [M_i, n_out] with unit inner stride");
  TORCH_CHECK(out.scalar_type() == (out_bf16 ? at::kBFloat16 : at::kFloat), "out dtype mismatch");
  TORCH_CHECK(p.out_stride < 0 || p.out_stride == out.stride(0), "all outputs must share the row stride");
  p.out_stride = out.stride(0);
  sg.out = reinterpret_cast<char*>(out.data_ptr());
}

// fp32 partial of segment s for the neighbour half of a split-K layer: the self half's output rows, whose columns are
// laid out like the output's (image i at i * N)
static void set_seg_part(SageParams& p, int s, const at::Tensor& t, int64_t M, int64_t n_out) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.dim() == 2 && t.size(0) == M && t.size(1) == n_out &&
              t.stride(1) == 1 && t.stride(0) >= (int64_t)p.n_imgs * p.N && t.stride(0) % 2 == 0 &&
              (reinterpret_cast<uintptr_t>(t.data_ptr()) & 7) == 0,
              "partial[i] must be an 8-byte aligned fp32 [M_i, n_out] view with an even row stride >= n_imgs * N");
  TORCH_CHECK(p.part_ld == 0 || p.part_ld == t.stride(0), "all partial views must share the row stride");
  p.part_ld = (int)t.stride(0);
  p.part[s] = t.data_ptr<float>();
}

// Multi-segment entry point.  All segments share the tables, the weight image, the bias and the output
// layout; segment i reads ids (self_vids[i], nbr_vids[i]) - or identity ids self_base[i] + m /
// nbr_base[i] + m*k + j when the tensors are None - and writes outs[i] ([M_i, n_out]) and optionally
// a_saves[i] ([M_i, K_total] bf16, the [self || agg] rows for the backward pass).
// ce = optional fused softmax cross-entropy on the output rows of segment 0:
//   [labels_table(int64), seeds(int64)|undefined, loss(fp32 >=1), dlogits(bf16 [M, stride]), dbias(fp32)|undefined]
// amax = [] or, for a max launch, one optional uint8 [M_i, >= d_nbr rounded up to 8] view per segment (a shared row
// stride, a multiple of 8): column c of row m receives the first neighbour j in [0, k_i) holding the maximum of column c
// drop_p > 0: inverted dropout with rate drop_p after bias and ReLU (a hidden layer's training forward): the mask of
// output element (drop_row0[i] + m, img * N + n) is a function of drop_state = {seed, step counter} (int64 [2], device),
// drop_layer and that position only (see dropout_bits); drop_p = 0 (the default) launches exactly as before
// split_half = 1 / 2: one half of a split-K layer, Z = x_self . W_self^T + agg . W_nbr^T, for a mean, sum or max layer
// whose padded K = 2 kp does not fit one launch.  w_img is the layer's images (2 kp / 64 k-blocks each) and a_saves[i]
// the [M_i, kp] views of the layer's [self || agg] rows that the half fills (row stride 2 kp).
//   1 (self half): ks all 0, outs[i] = the fp32 partial (no bias, ReLU, dropout, amax or CE)
//   2 (neighbour half): partial[i] = that partial, added to the accumulators before bias -> ReLU -> dropout -> store
void sage_fused_multi(const at::Tensor& tself_desc, const at::Tensor& tnbr_desc,
                      const std::vector<c10::optional<at::Tensor>>& self_vids,
                      const std::vector<c10::optional<at::Tensor>>& nbr_vids,
                      const std::vector<int64_t>& self_base, const std::vector<int64_t>& nbr_base,
                      const std::vector<int64_t>& Ms, const std::vector<int64_t>& ks,
                      const std::vector<at::Tensor>& outs, const std::vector<c10::optional<at::Tensor>>& a_saves,
                      int64_t mode, const at::Tensor& w_img, const c10::optional<at::Tensor>& bias, int64_t N,
                      int64_t n_out, bool relu, bool out_bf16,
                      const std::vector<c10::optional<at::Tensor>>& ce, int64_t ce_world, int64_t n_imgs,
                      const std::vector<c10::optional<at::Tensor>>& amax, const c10::optional<at::Tensor>& drop_state,
                      double drop_p, int64_t drop_layer, const std::vector<int64_t>& drop_row0, int64_t split_half,
                      const std::vector<c10::optional<at::Tensor>>& partial) {
  TORCH_CHECK(w_img.is_cuda() && w_img.scalar_type() == at::kBFloat16, "w_img must be CUDA bf16");
  TORCH_CHECK(mode >= kConcatMean && mode <= kConcatMax, "unknown aggregation mode ", mode);
  c10::cuda::CUDAGuard guard(w_img.device());
  const int nseg = (int)Ms.size();
  TORCH_CHECK(nseg >= 1 && nseg <= kMaxSegs, "1..", kMaxSegs, " segments per launch");
  TORCH_CHECK((int)ks.size() == nseg && (int)outs.size() == nseg && (int)a_saves.size() == nseg &&
              (int)self_vids.size() == nseg && (int)nbr_vids.size() == nseg && (int)self_base.size() == nseg &&
              (int)nbr_base.size() == nseg, "per-segment argument lists must have equal lengths");
  SageParams p;
  bool any_nbr = false;
  for (int s = 0; s < nseg; ++s) any_nbr = any_nbr || ks[s] > 0;
  if (split_half == 1)
    TORCH_CHECK(!any_nbr && ce.empty() && amax.empty() && drop_p == 0.0 && !relu && !out_bf16 && !(bias.has_value() && bias->defined()),
                "the self half of a split-K layer reads no neighbours (ks = 0) and writes the bare fp32 partial");
  if (split_half == 2) TORCH_CHECK(ce.empty(), "a split-K layer computes its loss outside the launch (no fused CE)");
  TORCH_CHECK(split_half == 2 ? (int)partial.size() == nseg : partial.empty(),
              "partial: one entry per segment of a neighbour-half launch, none otherwise");
  at::Tensor b;
  const size_t smem = init_layer_params(p, tself_desc, tnbr_desc, any_nbr, mode, w_img, bias, b, N, n_out, relu, out_bf16, n_imgs,
                                        split_half);
  p.nseg = nseg;
  {
    const int vec = p.tnbr.dtype == 0 ? 4 : 8;
    const int lanes_row = (p.kp_nbr > 0 ? p.kp_nbr : p.kp_self) / vec;
    const int rpi = lanes_row < 32 ? 32 / lanes_row : 1;
    for (int s = 0; s < nseg; ++s)
      TORCH_CHECK(rpi * (ks[s] + 1) <= kScrCap, "fan-out too large for the fused kernel's pointer scratch: k <= ", kScrCap / rpi - 1);
  }
  std::vector<at::Tensor> keep;
  const int k_total = p.kp_self + p.kp_nbr;
  p.out_stride = -1;
  for (int s = 0; s < nseg; ++s) {
    SageSeg& sg = p.seg[s];
    sg.M = (int)Ms[s]; sg.k = (int)ks[s];
    sg.self_base = self_base[s]; sg.nbr_base = nbr_base[s];
    if (self_vids[s].has_value() && self_vids[s]->defined()) {
      at::Tensor t = self_vids[s]->contiguous(); check_cuda_i64(t, "self_vids");
      TORCH_CHECK(t.numel() == Ms[s]); keep.push_back(t); sg.self_vids = t.data_ptr<int64_t>();
    }
    if (nbr_vids[s].has_value() && nbr_vids[s]->defined()) {
      at::Tensor t = nbr_vids[s]->contiguous(); check_cuda_i64(t, "nbr_vids");
      TORCH_CHECK(t.numel() == Ms[s] * ks[s]); keep.push_back(t); sg.nbr_vids = t.data_ptr<int64_t>();
    }
    set_seg_out(p, sg, outs[s], Ms[s], n_out, out_bf16);
    if (a_saves[s].has_value() && a_saves[s]->defined()) {
      const at::Tensor& a = *a_saves[s];
      const int64_t a_ld = split_half != 0 ? 2 * (int64_t)k_total : k_total;     // split-K: the layer's full rows
      TORCH_CHECK(a.scalar_type() == at::kBFloat16 && a.dim() == 2 && a.size(0) == Ms[s] && a.size(1) == k_total &&
                  a.stride(1) == 1 && a.stride(0) == a_ld, "a_saves[i] must be a bf16 [M_i, K_total] view with row stride ", a_ld);
      sg.a_save = reinterpret_cast<__nv_bfloat16*>(a.data_ptr());
      p.a_ld = (int)a_ld;
    }
    if (split_half == 2 && partial[s].has_value() && partial[s]->defined()) set_seg_part(p, s, *partial[s], Ms[s], n_out);
  }
  if (!amax.empty()) {
    TORCH_CHECK(mode == kConcatMax && (int)amax.size() == nseg, "amax needs a max launch and one entry per segment");
    for (int s = 0; s < nseg; ++s) {
      if (!(amax[s].has_value() && amax[s]->defined())) continue;
      const at::Tensor& a = *amax[s];
      TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kByte && a.dim() == 2 && a.size(0) == Ms[s] && a.stride(1) == 1 &&
                  a.size(1) >= (p.tnbr.dim + 7) / 8 * 8 && a.stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(a.data_ptr()) & 7) == 0,
                  "amax[i] must be an 8-byte aligned uint8 [M_i, >= d_nbr rounded up to 8] view, row stride a multiple of 8");
      TORCH_CHECK(ks[s] <= 256, "amax holds neighbour indices below 256");
      TORCH_CHECK(p.amax_ld == 0 || p.amax_ld == a.stride(0), "all amax views must share the row stride");
      p.amax_ld = (int)a.stride(0);
      p.amax[s] = reinterpret_cast<uint8_t*>(a.data_ptr());
    }
  }
  if (p.out_stride < 0) p.out_stride = n_out;
  TORCH_CHECK(drop_p >= 0.0 && drop_p < 1.0, "dropout rate must be in [0, 1), got ", drop_p);
  if (drop_p > 0.0) {
    TORCH_CHECK(drop_state.has_value() && drop_state->defined(), "dropout needs its {seed, counter} state");
    const at::Tensor& st = *drop_state;
    TORCH_CHECK(st.is_cuda() && st.scalar_type() == at::kLong && st.numel() == 2 && st.is_contiguous() &&
                (reinterpret_cast<uintptr_t>(st.data_ptr()) & 15) == 0, "drop_state must be a 16-byte aligned CUDA int64 [2]");
    TORCH_CHECK(ce.empty(), "dropout applies to hidden layers, not to the fused-CE top layer");
    TORCH_CHECK((int)drop_row0.size() == nseg, "drop_row0 needs one row offset per segment");
    TORCH_CHECK(drop_layer >= 0 && drop_layer < 256, "drop_layer must be in [0, 256)");
    p.drop_state = reinterpret_cast<const unsigned long long*>(st.data_ptr());
    p.drop_thr = (uint32_t)std::llround(drop_p * 65536.0);
    p.drop_scale = (float)(1.0 / (1.0 - drop_p));
    p.drop_layer = (uint32_t)drop_layer;
    for (int s = 0; s < nseg; ++s) {
      TORCH_CHECK(drop_row0[s] >= 0 && drop_row0[s] + Ms[s] <= (int64_t)INT32_MAX, "drop_row0 out of range");
      p.drop_row0[s] = (int)drop_row0[s];
    }
  }
  if (!ce.empty()) {
    TORCH_CHECK(ce.size() == 5 && nseg == 1 && N <= 64, "fused CE needs one segment and n_out <= 64");
    TORCH_CHECK(p.seg[0].out != nullptr && !out_bf16, "fused CE needs the fp32 logits output (its second phase re-reads it)");
    const at::Tensor& labels = *ce[0];
    TORCH_CHECK(labels.is_cuda() && labels.scalar_type() == at::kLong);
    p.ce_labels = labels.data_ptr<int64_t>();
    if (ce[1].has_value() && ce[1]->defined()) {
      TORCH_CHECK(ce[1]->scalar_type() == at::kLong && ce[1]->numel() == Ms[0] && ce[1]->is_contiguous());
      p.ce_seeds = ce[1]->data_ptr<int64_t>();
    } else {
      TORCH_CHECK(labels.numel() >= Ms[0]);
    }
    p.ce_world = (int)std::max<int64_t>(ce_world, 1);
    const at::Tensor& loss = *ce[2];
    TORCH_CHECK(loss.is_cuda() && loss.scalar_type() == at::kFloat && loss.numel() >= 1);
    p.ce_loss = loss.data_ptr<float>();
    const at::Tensor& dl = *ce[3];
    TORCH_CHECK(dl.is_cuda() && dl.scalar_type() == at::kBFloat16 && dl.dim() == 2 && dl.size(0) == Ms[0] && dl.stride(1) == 1 &&
                dl.stride(0) >= n_out, "dlogits must be bf16 [M, >= n_out]");
    p.ce_dlogits = reinterpret_cast<__nv_bfloat16*>(dl.data_ptr());
    p.ce_dl_stride = (int)dl.stride(0);
    if (ce[4].has_value() && ce[4]->defined()) {
      TORCH_CHECK(ce[4]->scalar_type() == at::kFloat && ce[4]->numel() >= n_out);
      p.ce_dbias = ce[4]->data_ptr<float>();
    }
    p.ce_inv_b = 1.f / (float)Ms[0];
  }
  p.dbg = g_dbg_ptr;
  plan_tiles(p);
  launch_persist(p, smem, at::cuda::getCurrentCUDAStream(), false, split_half != 0);
}

// Layer-wise full-neighbourhood inference: ONE layer over every row of a CSR (row m of `out` aggregates the neighbour
// rows csr_indices[csr_indptr[m] .. csr_indptr[m + 1]) of tnbr; its self row is self_vids[m] in tself).
// hubs = [] or [hub_map int32 [M] (-1 = ordinary row), hub_cptr int32 [n_hub + 1], chunks int64 [n_chunks, 2]
// (edge ranges), part fp32 [>= n_chunks * kp_nbr]]: the hub rows' adjacency chunks are first summed into `part` by
// sage_hub_partial_kernel.  plan_deg = mean degree of the ordinary rows (tile costing).
// split_half = 2: the neighbour half of a split-K layer (see sage_fused_multi), which adds `partial` (fp32 [M, n_out],
// the self half's output over the same rows) before the epilogue.
void sage_fused_csr(const at::Tensor& tself_desc, const at::Tensor& tnbr_desc, const at::Tensor& self_vids,
                    const at::Tensor& csr_indptr, const at::Tensor& csr_indices, const std::vector<at::Tensor>& hubs,
                    const at::Tensor& out, int64_t mode, const at::Tensor& w_img, const c10::optional<at::Tensor>& bias,
                    int64_t N, int64_t n_out, bool relu, bool out_bf16, int64_t n_imgs, int64_t plan_deg, int64_t split_half,
                    const c10::optional<at::Tensor>& partial) {
  TORCH_CHECK(split_half == 0 || split_half == 2, "the CSR mode runs a whole layer or the neighbour half of a split-K layer");
  TORCH_CHECK((split_half == 2) == (partial.has_value() && partial->defined()), "the neighbour half needs the self half's partial");
  TORCH_CHECK(w_img.is_cuda() && w_img.scalar_type() == at::kBFloat16, "w_img must be CUDA bf16");
  c10::cuda::CUDAGuard guard(w_img.device());
  TORCH_CHECK(mode >= kConcatMean && mode <= kConcatMax, "unknown aggregation mode ", mode);
  const int64_t M = self_vids.numel();
  check_cuda_i64(self_vids, "self_vids");
  check_cuda_i64(csr_indptr, "csr_indptr");
  check_cuda_i64(csr_indices, "csr_indices");
  TORCH_CHECK(self_vids.is_contiguous() && csr_indptr.is_contiguous() && csr_indices.is_contiguous(), "CSR operands must be contiguous");
  TORCH_CHECK(csr_indptr.numel() == M + 1, "csr_indptr must have M + 1 entries");
  TORCH_CHECK(M < (int64_t)INT32_MAX, "too many rows");
  SageParams p;
  at::Tensor b;
  const size_t smem = init_layer_params(p, tself_desc, tnbr_desc, true, mode, w_img, bias, b, N, n_out, relu, out_bf16, n_imgs,
                                        split_half);
  p.nseg = 1;
  SageSeg& sg = p.seg[0];
  sg.M = (int)M;
  sg.k = (int)std::max<int64_t>(plan_deg, 1);        // tile costing only: the CSR gather reads the row's own degree
  sg.self_vids = self_vids.data_ptr<int64_t>();
  p.out_stride = -1;
  set_seg_out(p, sg, out, M, n_out, out_bf16);
  TORCH_CHECK(sg.out != nullptr, "CSR mode needs an output");
  if (split_half == 2) set_seg_part(p, 0, *partial, M, n_out);
  p.csr_indptr = csr_indptr.data_ptr<int64_t>();
  p.csr_indices = csr_indices.data_ptr<int64_t>();
  const cudaStream_t stream = at::cuda::getCurrentCUDAStream();
  if (!hubs.empty()) {
    TORCH_CHECK(hubs.size() == 4, "hubs = [hub_map, hub_cptr, chunks, part]");
    const at::Tensor &hmap = hubs[0], &cptr = hubs[1], &chunks = hubs[2], &part = hubs[3];
    TORCH_CHECK(hmap.is_cuda() && hmap.scalar_type() == at::kInt && hmap.numel() == M && hmap.is_contiguous(), "hub_map must be int32 [M]");
    TORCH_CHECK(cptr.is_cuda() && cptr.scalar_type() == at::kInt && cptr.is_contiguous() && cptr.numel() >= 1, "hub_cptr must be int32");
    check_cuda_i64(chunks, "chunks");
    TORCH_CHECK(chunks.is_contiguous() && chunks.dim() == 2 && chunks.size(1) == 2, "chunks must be int64 [n_chunks, 2]");
    const int64_t n_chunks = chunks.size(0);
    TORCH_CHECK(n_chunks * 128 < (int64_t)INT32_MAX, "too many hub chunks");
    TORCH_CHECK(part.is_cuda() && part.scalar_type() == at::kFloat && part.is_contiguous() && part.numel() >= n_chunks * p.kp_nbr,
                "part must be fp32 [>= n_chunks * kp_nbr]");
    TORCH_CHECK((reinterpret_cast<uintptr_t>(part.data_ptr()) & 15) == 0, "part must be 16 B aligned");
    p.hub_map = hmap.data_ptr<int>();
    p.hub_cptr = cptr.data_ptr<int>();
    p.hub_part = part.data_ptr<float>();
    p.hub_stride = p.kp_nbr;
    if (n_chunks > 0) {
      const int vec = p.tnbr.dtype == 0 ? 4 : 8;
      const int lanes_row = p.kp_nbr / vec;
      const int64_t warps = n_chunks * (lanes_row > 32 ? lanes_row / 32 : 1);
      const unsigned grid = (unsigned)((warps * 32 + 255) / 256);
      const int64_t* ch = chunks.data_ptr<int64_t>();
      float* pt = part.data_ptr<float>();
      // max: partial maxima; mean, sum and gcn: partial sums
#define HUB_LAUNCH(DT, MX) sage_hub_partial_kernel<kCsrU, DT, MX><<<grid, 256, 0, stream>>>( \
          p.tnbr, p.wshift_nbr, p.csr_indices, ch, (int)n_chunks, p.kp_nbr, pt, p.zero_row)
      const bool mx = mode == kConcatMax;
      if (p.tnbr.dtype == 0) { if (mx) HUB_LAUNCH(0, true); else HUB_LAUNCH(0, false); }
      else if (p.tnbr.dtype == 1) { if (mx) HUB_LAUNCH(1, true); else HUB_LAUNCH(1, false); }
      else { if (mx) HUB_LAUNCH(2, true); else HUB_LAUNCH(2, false); }
#undef HUB_LAUNCH
      C10_CUDA_KERNEL_LAUNCH_CHECK();
    }
  }
  p.dbg = g_dbg_ptr;
  plan_tiles(p);
  launch_persist(p, smem, stream, true, split_half != 0);
}

// single-segment convenience wrapper (autograd op in ops/sage.py)
std::vector<at::Tensor> sage_fused_forward(const at::Tensor& tself_desc,
                                           const c10::optional<at::Tensor>& self_vids,
                                           const at::Tensor& tnbr_desc,
                                           const c10::optional<at::Tensor>& nbr_vids, int64_t M,
                                           int64_t k, int64_t mode, const at::Tensor& w_img,
                                           const c10::optional<at::Tensor>& bias, int64_t N,
                                           int64_t n_out, bool relu, bool out_bf16, bool save_a) {
  c10::cuda::CUDAGuard guard(w_img.device());
  auto opts = w_img.options();
  at::Tensor out = at::empty({M, n_out}, opts.dtype(out_bf16 ? at::kBFloat16 : at::kFloat));
  at::Tensor a_save;
  if (save_a) {
    const TableView ts = table_from_desc(tself_desc), tn = table_from_desc(tnbr_desc);
    const int64_t k_total = ((mode == kGcnMean) ? 0 : pad_k(ts.dim)) + (k > 0 ? pad_k(tn.dim) : 0);
    a_save = at::empty({M, k_total}, opts.dtype(at::kBFloat16));
  }
  if (M == 0) return {out, a_save};
  sage_fused_multi(tself_desc, tnbr_desc, {self_vids}, {nbr_vids}, {0}, {0}, {M}, {k}, {out},
                   {save_a ? c10::optional<at::Tensor>(a_save) : c10::nullopt}, mode, w_img, bias, N, n_out, relu, out_bf16,
                   {}, 1, 1, {}, c10::nullopt, 0.0, 0, {}, 0, {});
  return {out, a_save};
}

// K7 standalone: out = act(A . W^T + b) for a dense bf16 A [M, K] (K multiple of 64, <= 512; N <= 256)
// on the same persistent wgmma kernel (the "gather" degenerates to staging A's rows).
at::Tensor tc_linear_forward(const at::Tensor& a, const at::Tensor& w_img, const c10::optional<at::Tensor>& bias,
                             int64_t N, int64_t n_out, bool relu, bool out_bf16) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kBFloat16 && a.dim() == 2 && a.stride(1) == 1,
              "A must be a CUDA bf16 [M, K] matrix with unit inner stride");
  const int64_t M = a.size(0), K = a.size(1);
  TORCH_CHECK(K % 8 == 0 && K >= 8 && K <= 512 && a.stride(0) % 8 == 0, "K must be a multiple of 8 in [8, 512]");
  c10::cuda::CUDAGuard guard(a.device());
  auto out = at::empty({M, n_out}, a.options().dtype(out_bf16 ? at::kBFloat16 : at::kFloat));
  if (M == 0) return out;
  std::vector<int64_t> d(4 + 2 * kMaxWorld, 0);
  d[0] = 1; d[1] = K; d[2] = a.stride(0); d[3] = 1; d[4] = M; d[4 + kMaxWorld] = reinterpret_cast<int64_t>(a.data_ptr());
  at::Tensor desc = at::from_blob(d.data(), {(int64_t)d.size()}, at::kLong).clone();
  sage_fused_multi(desc, desc, {c10::nullopt}, {c10::nullopt}, {0}, {0}, {M}, {0}, {out}, {c10::nullopt}, kConcatMean, w_img, bias,
                   N, n_out, relu, out_bf16, {}, 1, 1, {}, c10::nullopt, 0.0, 0, {}, 0, {});
  return out;
}

}  // namespace glb
