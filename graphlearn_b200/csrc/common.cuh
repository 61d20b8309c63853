// Common device-side utilities for the graphlearn_b200 sm_90a kernels.
//
// * PeerTable   — by-value table of per-rank base pointers (NVLink P2P / IPC
//                 mapped).  Every sharded array (CSR indptr/indices, feature
//                 tables, ...) is addressed as table.p[owner] + row*stride so
//                 that a kernel dereferences peer HBM directly; this replaces
//                 the reference's Partition -> gRPC -> Stitch round trip
//                 (graphlearn/src/core/runner/op_runner.h:60-152).
// * Philox4x32  — counter based RNG so that (seed, step, op, element) fully
//                 determines a draw: reproducible samplers and resumable
//                 checkpoints (SURVEY §7.4 item 4).
// * vid         — "virtual id" = row * world + owner.  With the reference's
//                 hash partitioning owner = |id| % world
//                 (graphlearn/src/core/partition/hash_partitioner.h:90-92);
//                 for dense id spaces vid == id.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cstdint>

namespace glb {

constexpr int kMaxWorld = 8;

struct PeerTable {
  const void* p[kMaxWorld];
};

struct PeerTableMut {
  void* p[kMaxWorld];
};

__host__ __device__ __forceinline__ int vid_owner(int64_t vid, int world) {
  return (int)(vid % world);
}
__host__ __device__ __forceinline__ int64_t vid_row(int64_t vid, int world) {
  return vid / world;
}

// ----------------------------------------------------------------------------
// Philox4x32-10
// ----------------------------------------------------------------------------
struct Philox {
  uint32_t key0, key1;
  __host__ __device__ __forceinline__ Philox(uint64_t seed)
      : key0((uint32_t)seed), key1((uint32_t)(seed >> 32)) {}

  __host__ __device__ __forceinline__ static void mulhilo(uint32_t a, uint32_t b,
                                                           uint32_t& hi, uint32_t& lo) {
#ifdef __CUDA_ARCH__
    lo = a * b;
    hi = __umulhi(a, b);
#else
    uint64_t p = (uint64_t)a * b;
    lo = (uint32_t)p;
    hi = (uint32_t)(p >> 32);
#endif
  }

  // counter = (c0,c1,c2,c3); returns 4 x 32 random bits
  __host__ __device__ __forceinline__ uint4 operator()(uint32_t c0, uint32_t c1,
                                                        uint32_t c2, uint32_t c3) const {
    uint32_t k0 = key0, k1 = key1;
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      uint32_t hi0, lo0, hi1, lo1;
      mulhilo(0xD2511F53u, c0, hi0, lo0);
      mulhilo(0xCD9E8D57u, c2, hi1, lo1);
      uint32_t n0 = hi1 ^ c1 ^ k0;
      uint32_t n1 = lo1;
      uint32_t n2 = hi0 ^ c3 ^ k1;
      uint32_t n3 = lo0;
      c0 = n0; c1 = n1; c2 = n2; c3 = n3;
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
  }
};

// RNG state lives in device memory so that CUDA-graph replays see fresh
// randomness: state[0] = seed, state[1] = step offset (bumped by a 1-thread
// kernel once per step).
struct RngState {
  uint64_t seed;
  uint64_t offset;
};

__device__ __forceinline__ uint4 rng4(const uint64_t* __restrict__ state, uint32_t op_salt,
                                       uint64_t elem) {
  uint64_t seed = state[0];
  uint64_t off = state[1];
  Philox ph(seed);
  return ph((uint32_t)elem, (uint32_t)(elem >> 32), (uint32_t)off,
            (uint32_t)(off >> 32) ^ (op_salt * 0x9E3779B9u));
}

// uniform integer in [0, n) from 32 random bits (Lemire multiply-shift; the
// bias is < n / 2^32 which is negligible for adjacency degrees).
__host__ __device__ __forceinline__ uint32_t bounded(uint32_t r, uint32_t n) {
#ifdef __CUDA_ARCH__
  return __umulhi(r, n);
#else
  return (uint32_t)(((uint64_t)r * n) >> 32);
#endif
}
__host__ __device__ __forceinline__ uint64_t bounded64(uint32_t r0, uint32_t r1, uint64_t n) {
  if (n <= 0xFFFFFFFFull) return bounded(r0, (uint32_t)n);
  uint64_t r = ((uint64_t)r0 << 32) | r1;
#ifdef __CUDA_ARCH__
  return __umul64hi(r, n);
#else
  return (uint64_t)(((unsigned __int128)r * n) >> 64);
#endif
}
__host__ __device__ __forceinline__ float u01(uint32_t r) {
  // (0,1]-open-left uniform
  return ((float)(r >> 8) + 0.5f) * (1.0f / 16777216.0f);
}

// ----------------------------------------------------------------------------
// Keyed bijection on [0, n): 4-round Feistel network on ceil(log2 n) bits with
// cycle walking.  Used for sampling WITHOUT replacement fully in parallel:
// slot j of row r takes element perm_r(j), all distinct by construction
// (reference semantic: graphlearn/src/core/operator/sampler/
// random_without_replacement_sampler.cc:59-68 shuffles an iota).
// ----------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

__host__ __device__ __forceinline__ uint32_t feistel_perm(uint32_t idx, uint32_t n,
                                                           uint32_t k0, uint32_t k1) {
  if (n <= 1) return 0;
#ifdef __CUDA_ARCH__
  int bits = 32 - __clz(n - 1);
#else
  int bits = 32 - __builtin_clz(n - 1);
#endif
  if (bits & 1) bits++;          // balanced halves => provable bijection
  if (bits < 2) bits = 2;
  const int hb = bits / 2;
  const uint32_t mask = (1u << hb) - 1;
  uint32_t x = idx;
  // cycle walking: domain 2^bits < 8n, expected < 8 iterations.  Walking the
  // cycle of a bijection of [0,2^bits) until we re-enter [0,n) is itself a
  // bijection of [0,n).
  for (int iter = 0; iter < 512; ++iter) {
    uint32_t l = x >> hb, r = x & mask;
#pragma unroll
    for (int round = 0; round < 4; ++round) {
      uint32_t f = mix32(r ^ (k0 + (uint32_t)round * 0x9E3779B9u)) ^ k1;
      uint32_t t = l ^ (f & mask);
      l = r; r = t;
    }
    x = (l << hb) | r;
    if (x < n) return x;
  }
  return idx % n;  // unreachable in practice (p < 0.875^512)
}

// ----------------------------------------------------------------------------
// misc
// ----------------------------------------------------------------------------
__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}
__device__ __forceinline__ uint2 ld_nc_u2(const uint2* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];"
               : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
__device__ __forceinline__ uint4 ld_nc_u4(const uint4* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}

__device__ __forceinline__ uint32_t ld_nc_u16(const uint16_t* p) {
  uint16_t r;
  asm volatile("ld.global.nc.L1::no_allocate.u16 %0, [%1];" : "=h"(r) : "l"(p));
  return (uint32_t)r;
}
// two e4m3 values (low byte first) -> fp32 pair
__device__ __forceinline__ float2 e4m3x2_to_float2(uint32_t two_bytes) {
  uint32_t h2;
  const uint16_t in = (uint16_t)two_bytes;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h2) : "h"(in));
  return __half22float2(*reinterpret_cast<__half2*>(&h2));
}

__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  // bf16 -> fp32 is a 16-bit shift: one SHL for the low element, one LOP for the high one (the library's
  // __bfloat1622float2 spends PRMT + shift on the high half)
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}

}  // namespace glb
