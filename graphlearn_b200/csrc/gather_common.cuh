// Row-gather helpers shared by the fused SAGE kernel (sage_fused.cu) and the attention kernels (gat.cu):
// raw 16-byte row chunks, vid -> (owner, row) locators and row addresses in local HBM / peer HBM / the replica cache.
#pragma once
#include "common.cuh"
#include "host_utils.h"

namespace glb {

// One 16-byte storage chunk of a feature row: 4 fp32 or 8 bf16 features.  Kept RAW
// (unconverted) so that a whole batch of row loads is issued back to back before the first use.
template <int DT> struct Chunk;
template <> struct Chunk<0> {
  static constexpr int kVec = 4;
  float4 v;
  __device__ __forceinline__ void load(const char* p) { v = ld_nc_f4(reinterpret_cast<const float4*>(p)); }
  __device__ __forceinline__ void add_to(float (&a)[4]) const { a[0] += v.x; a[1] += v.y; a[2] += v.z; a[3] += v.w; }
  __device__ __forceinline__ void get(float (&a)[4]) const { a[0] = v.x; a[1] = v.y; a[2] = v.z; a[3] = v.w; }
};
template <> struct Chunk<1> {
  static constexpr int kVec = 8;
  uint4 v;
  __device__ __forceinline__ void load(const char* p) { v = ld_nc_u4(reinterpret_cast<const uint4*>(p)); }
  __device__ __forceinline__ void add_to(float (&a)[8]) const {
    float2 x;
    x = unpack_bf16x2(v.x); a[0] += x.x; a[1] += x.y;
    x = unpack_bf16x2(v.y); a[2] += x.x; a[3] += x.y;
    x = unpack_bf16x2(v.z); a[4] += x.x; a[5] += x.y;
    x = unpack_bf16x2(v.w); a[6] += x.x; a[7] += x.y;
  }
  __device__ __forceinline__ void get(float (&a)[8]) const {
    float2 x;
    x = unpack_bf16x2(v.x); a[0] = x.x; a[1] = x.y;
    x = unpack_bf16x2(v.y); a[2] = x.x; a[3] = x.y;
    x = unpack_bf16x2(v.z); a[4] = x.x; a[5] = x.y;
    x = unpack_bf16x2(v.w); a[6] = x.x; a[7] = x.y;
  }
};

// fp8 (e4m3) rows with one bf16 scale per 32-element block: a chunk is 8 elements = 8 bytes + the block's scale
template <> struct Chunk<2> {
  static constexpr int kVec = 8;
  uint2 v;
  float s;
  __device__ __forceinline__ void load_row(const char* row, int chunk, int scale_off) {
    v = ld_nc_u2(reinterpret_cast<const uint2*>(row) + chunk);
    s = __uint_as_float(ld_nc_u16(reinterpret_cast<const uint16_t*>(row + scale_off) + (chunk >> 2)) << 16);
  }
  __device__ __forceinline__ void add_to(float (&a)[8]) const {
    float2 x;
    x = e4m3x2_to_float2(v.x);       a[0] = fmaf(x.x, s, a[0]); a[1] = fmaf(x.y, s, a[1]);
    x = e4m3x2_to_float2(v.x >> 16); a[2] = fmaf(x.x, s, a[2]); a[3] = fmaf(x.y, s, a[3]);
    x = e4m3x2_to_float2(v.y);       a[4] = fmaf(x.x, s, a[4]); a[5] = fmaf(x.y, s, a[5]);
    x = e4m3x2_to_float2(v.y >> 16); a[6] = fmaf(x.x, s, a[6]); a[7] = fmaf(x.y, s, a[7]);
  }
  __device__ __forceinline__ void get(float (&a)[8]) const {     // dequantised
    float2 x;
    x = e4m3x2_to_float2(v.x);       a[0] = x.x * s; a[1] = x.y * s;
    x = e4m3x2_to_float2(v.x >> 16); a[2] = x.x * s; a[3] = x.y * s;
    x = e4m3x2_to_float2(v.y);       a[4] = x.x * s; a[5] = x.y * s;
    x = e4m3x2_to_float2(v.y >> 16); a[6] = x.x * s; a[7] = x.y * s;
  }
};

// uniform loader: 16-byte chunk `chunk` of a fp32 / bf16 row, or 8-element chunk + block scale of an fp8 row
template <int DT>
__device__ __forceinline__ void load_chunk(Chunk<DT>& c, const char* row, int chunk, int scale_off) {
  if constexpr (DT == 2) c.load_row(row, chunk, scale_off);
  else c.load(row + (size_t)chunk * 16);
}

// locator of a table row packed into 32 bits: (row << 3) | owner, 0xFFFFFFFF = missing
__device__ __forceinline__ uint32_t make_loc(const TableView& t, int64_t vid, int wshift) {
  if (vid < 0) return 0xFFFFFFFFu;
  int owner; int64_t row;
  if (wshift >= 0) { owner = (int)(vid & ((1 << wshift) - 1)); row = vid >> wshift; }
  else { owner = (int)(vid % t.world); row = vid / t.world; }
  if (row >= t.nrows[owner]) return 0xFFFFFFFFu;
  return ((uint32_t)row << 3) | (uint32_t)owner;
}
__device__ __forceinline__ const char* loc_ptr(const TableView& t, uint32_t loc, uint32_t row_bytes) {
  return reinterpret_cast<const char*>(t.base.p[loc & 7u]) + (size_t)(loc >> 3) * row_bytes;
}

// row address of a vid: the local replica-cache copy when the row is remote and cached (N17),
// the owner's HBM otherwise; `zero_row` for missing / padded ids
__device__ __forceinline__ const char* vid_ptr(const TableView& t, int64_t vid, int wshift, uint32_t row_bytes,
                                               const char* zero_row) {
  const uint32_t loc = make_loc(t, vid, wshift);
  if (loc == 0xFFFFFFFFu) return zero_row;
  if (t.cmap != nullptr && (int)(loc & 7u) != t.self) {
    const int s = __ldg(t.cmap + vid);
    if (s >= 0) return t.cbase + (size_t)s * row_bytes;
  }
  return loc_ptr(t, loc, row_bytes);
}

}  // namespace glb
