// K10: brute-force KNN as ONE kernel per 128-query tile - score GEMM on wgmma with a fused running top-k,
// the [B, N] score matrix is never materialised.
//
//   scores[q, x] = <Q[q], X[x]>            (inner product)      or      2 <Q[q], X[x]> - |X[x]|^2     (L2; larger = closer)
//
// Every CTA (one per SM) owns a contiguous range of database rows and walks it in slabs of 128 rows:
//   warps 4..11  producers : database rows (fp32 or bf16, optionally through a row-index list = an IVF inverted
//                            list) -> bf16 -> K-major SWIZZLE_128B operand tile in shared memory (double buffered)
//   warps 0..3   MMA+top-k : one warpgroup computes D[128 queries x 32 rows] = Q . X^T slice by slice with wgmma
//                            (two M=64 halves, fp32 accumulators in registers), parks the slice in shared memory, and
//                            then one thread per query scans its 32 scores and keeps the k best (value, row) in shared
//                            memory behind a register-held admission threshold
// The per-CTA lists are merged by knn_merge_kernel (one warp per query), which also reads the partial lists of PEER GPUs
// straight from their HBM (the reference broadcasts the query to every server and merges with a k-heap over gRPC:
// graphlearn/src/contrib/knn/knn_request.cc:96-111,167-202; index types: index_factory.cc:28-50).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cfloat>
#include <cstring>
#include "host_utils.h"
#include "gmma.cuh"

namespace glb {

constexpr int kKnnQ = 128;                 // queries per tile (two wgmma M = 64 halves)
constexpr int kKnnSlab = 128;              // database rows per slab
constexpr int kKnnSlice = 32;              // database rows per MMA slice (wgmma N)
constexpr int kKnnScoreLd = kKnnSlice + 1; // row pitch of the staged score slice (conflict-free per-query reads)
constexpr int kKnnTopWarps = 4, kKnnProdWarp0 = 4, kKnnProdWarps = 8;
constexpr int kKnnThreads = (kKnnProdWarp0 + kKnnProdWarps) * 32;   // 384
constexpr int kKnnMaxK = 64;

struct KnnParams {
  const void* x; int x_dtype; int64_t x_stride;     // local shard rows (0 fp32 / 1 bf16), stride in elements
  const float* x_norm;                               // |x|^2 per row (L2) or null (inner product)
  const int64_t* row_list;                           // optional: scan x[row_list[i]] for i in [0, n)   (IVF list)
  int64_t n;                                         // rows to scan
  const __nv_bfloat16* q;                            // [128, dpad] bf16, zero padded (rows >= B are zero)
  int dpad, dim, k, B;
  float* out_s;                                      // [grid, 128, k] partial scores
  int64_t* out_i;                                    // [grid, 128, k] partial row indices (into x / row_list space)
  int64_t rows_per_cta;
  int n_xbuf;                                        // database slab buffers: 2 (double buffered) or 1 when two do not fit
};

__global__ void __launch_bounds__(kKnnThreads, 1) knn_flat_kernel(const __grid_constant__ KnnParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (gmma::smem_u32(smem_raw) & 1023u)) & 1023u);
  const int nkb = p.dpad >> 6;
  const uint32_t tile_bytes = (uint32_t)nkb * (128 * 128);
  uint8_t* sQ = smem;
  uint8_t* sX = sQ + tile_bytes;                                   // [n_xbuf] slabs
  float* sNorm = reinterpret_cast<float*>(sX + (size_t)p.n_xbuf * tile_bytes);   // [n_xbuf][128]
  float* sScore = sNorm + p.n_xbuf * kKnnSlab;                     // [128][kKnnScoreLd] one score slice
  float* topv = sScore + kKnnQ * kKnnScoreLd;                      // [k][128]
  int* topi = reinterpret_cast<int*>(topv + (size_t)p.k * kKnnQ);  // [k][128]  (slab-relative global index as int)
  uint64_t* bars = reinterpret_cast<uint64_t*>(topi + (size_t)p.k * kKnnQ);
  uint64_t* x_full = bars;          // [2] producers -> MMA
  uint64_t* x_free = bars + 2;      // [2] MMA / top-k -> producers (operand tile and norm slice consumed)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t r_begin = (int64_t)blockIdx.x * p.rows_per_cta;
  const int64_t r_end = min(p.n, r_begin + p.rows_per_cta);
  const int n_slabs = r_end > r_begin ? (int)((r_end - r_begin + kKnnSlab - 1) / kKnnSlab) : 0;

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) {
      gmma::mbar_init(x_full + i, kKnnProdWarps);
      gmma::mbar_init(x_free + i, kKnnTopWarps);
    }
    gmma::fence_barrier_init();
  }
  // query tile -> SW128 K-major (all threads), top-k lists cleared
  {
    const int chunks_row = p.dpad >> 3;
    for (int i = tid; i < kKnnQ * chunks_row; i += kKnnThreads) {
      const int r = i / chunks_row, c = i - r * chunks_row;
      const uint4 v = *reinterpret_cast<const uint4*>(p.q + (size_t)r * p.dpad + c * 8);
      const int kcol = c * 8;
      *reinterpret_cast<uint4*>(sQ + (size_t)(kcol >> 6) * (128 * 128) + gmma::sw128_offset((uint32_t)r, (uint32_t)(kcol & 63))) = v;
    }
    for (int i = tid; i < p.k * kKnnQ; i += kKnnThreads) { topv[i] = -FLT_MAX; topi[i] = -1; }
  }
  gmma::fence_proxy_async_smem();
  __syncthreads();

  if (warp < kKnnTopWarps) {
    // ------------------------------------------------------------------ score MMA + running top-k (thread = query)
    const int q = warp * 32 + lane;
    float thr = -FLT_MAX;                                   // smallest kept score (admission threshold)
    int thr_pos = 0;
    const uint32_t q_base = gmma::smem_u32(sQ);
    for (int s = 0; s < n_slabs; ++s) {
      const int b = s % p.n_xbuf;
      gmma::mbar_wait(x_full + b, (uint32_t)((s / p.n_xbuf) & 1));
      const int64_t base = r_begin + (int64_t)s * kKnnSlab;
      const int valid = (int)min((int64_t)kKnnSlab, r_end - base);
      const uint32_t x_base = gmma::smem_u32(sX + (size_t)b * tile_bytes);
      for (int c0 = 0; c0 < valid; c0 += kKnnSlice) {
#pragma unroll
        for (int mh = 0; mh < 2; ++mh) {
          float d[16];
          gmma::wgmma_fence();
          for (int kb = 0; kb < nkb; ++kb) {
            const uint32_t a_kb = q_base + (uint32_t)kb * (128 * 128) + (uint32_t)mh * (64 * 128);
            const uint32_t b_kb = x_base + (uint32_t)kb * (128 * 128) + (uint32_t)c0 * 128;
#pragma unroll
            for (int k4 = 0; k4 < 4; ++k4)
              gmma::mma_m64n32_bf16<0, 0>(d, gmma::make_desc_sw128(a_kb + k4 * 32), gmma::make_desc_sw128(b_kb + k4 * 32), (kb | k4) ? 1u : 0u);
          }
          gmma::wgmma_commit();
          gmma::wgmma_wait<0>();
          gmma::fence_regs(d);
          const int r = mh * 64 + warp * 16 + (lane >> 2);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            sScore[r * kKnnScoreLd + c] = d[4 * j];
            sScore[r * kKnnScoreLd + c + 1] = d[4 * j + 1];
            sScore[(r + 8) * kKnnScoreLd + c] = d[4 * j + 2];
            sScore[(r + 8) * kKnnScoreLd + c + 1] = d[4 * j + 3];
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kKnnTopWarps * 32) : "memory");     // the slice's scores are staged
        if (q < p.B) {
          for (int i = 0; i < kKnnSlice; ++i) {
            if (c0 + i < valid) {
              float sc = sScore[q * kKnnScoreLd + i];
              if (p.x_norm) sc = 2.f * sc - sNorm[b * kKnnSlab + c0 + i];
              if (sc > thr) {
                topv[thr_pos * kKnnQ + q] = sc;
                topi[thr_pos * kKnnQ + q] = (int)(base + c0 + i - r_begin);
                thr = FLT_MAX;
                for (int j = 0; j < p.k; ++j) {             // new minimum of the kept set
                  const float t = topv[j * kKnnQ + q];
                  if (t < thr) { thr = t; thr_pos = j; }
                }
              }
            }
          }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kKnnTopWarps * 32) : "memory");     // the staging slice may be overwritten
      }
      __syncwarp();
      if (lane == 0) gmma::mbar_arrive(x_free + b);
    }
    // publish this CTA's list
    if (q < p.B) {
      float* os = p.out_s + ((size_t)blockIdx.x * kKnnQ + q) * p.k;
      int64_t* oi = p.out_i + ((size_t)blockIdx.x * kKnnQ + q) * p.k;
      for (int j = 0; j < p.k; ++j) {
        const int li = topi[j * kKnnQ + q];
        os[j] = topv[j * kKnnQ + q];
        oi[j] = li < 0 ? -1 : (p.row_list ? p.row_list[r_begin + li] : r_begin + li);
      }
    }
  } else {
    // ------------------------------------------------------------------ producers: database slab -> bf16 SW128 tile
    const int pt = tid - kKnnProdWarp0 * 32;                 // 0..255
    const int chunks_row = p.dpad >> 3;                      // 16-byte bf16 chunks per row
    const int per_slab = kKnnSlab * chunks_row;
    for (int s = 0; s < n_slabs; ++s) {
      const int b = s % p.n_xbuf;
      gmma::mbar_wait(x_free + b, (uint32_t)(((s / p.n_xbuf) & 1) ^ 1));     // MMA and top-k are done with the tile and norm slice
      const int64_t base = r_begin + (int64_t)s * kKnnSlab;
      uint8_t* dst = sX + (size_t)b * tile_bytes;
      // batches of 8 chunks per thread: all loads of a batch are issued before the first store (one DRAM round trip per
      // batch instead of one per chunk - the slab loop is latency bound otherwise)
      constexpr int kPB = 8, kPT = kKnnProdWarps * 32;
      for (int i0 = pt; i0 < per_slab; i0 += kPB * kPT) {
        uint4 vals[kPB];
#pragma unroll
        for (int u = 0; u < kPB; ++u) {
          const int i = i0 + u * kPT;
          uint4 val = make_uint4(0u, 0u, 0u, 0u);
          if (i < per_slab) {
            const int r = i / chunks_row, c = i - r * chunks_row;
            const int64_t li = base + r;
            if (li < r_end && c * 8 < p.dim) {
              const int64_t row = p.row_list ? __ldg(p.row_list + li) : li;
              if (p.x_dtype == 1) {
                val = ld_nc_u4(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.x) + row * p.x_stride) + c);
                if (c * 8 + 8 > p.dim) {                          // mask the tail beyond the real dimension
                  __nv_bfloat16* e = reinterpret_cast<__nv_bfloat16*>(&val);
                  for (int j = 0; j < 8; ++j) if (c * 8 + j >= p.dim) e[j] = __float2bfloat16(0.f);
                }
              } else {
                const float* src = reinterpret_cast<const float*>(p.x) + row * p.x_stride + c * 8;
                float f[8];
#pragma unroll
                for (int j = 0; j < 8; ++j) f[j] = (c * 8 + j < p.dim) ? __ldg(src + j) : 0.f;
                val.x = pack_bf16x2(f[0], f[1]); val.y = pack_bf16x2(f[2], f[3]); val.z = pack_bf16x2(f[4], f[5]); val.w = pack_bf16x2(f[6], f[7]);
              }
            }
          }
          vals[u] = val;
        }
#pragma unroll
        for (int u = 0; u < kPB; ++u) {
          const int i = i0 + u * kPT;
          if (i < per_slab) {
            const int r = i / chunks_row, c = i - r * chunks_row;
            const int kcol = c * 8;
            *reinterpret_cast<uint4*>(dst + (size_t)(kcol >> 6) * (128 * 128) + gmma::sw128_offset((uint32_t)r, (uint32_t)(kcol & 63))) = vals[u];
          }
        }
      }
      if (p.x_norm && pt < kKnnSlab) {
        const int64_t li = base + pt;
        sNorm[b * kKnnSlab + pt] = li < r_end ? __ldg(p.x_norm + (p.row_list ? __ldg(p.row_list + li) : li)) : 0.f;
      }
      gmma::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) gmma::mbar_arrive(x_full + b);
    }
  }
}

// k-way merge: one warp per query selects the k best of all candidate lists - the partial lists of this GPU's CTAs or
// the per-rank lists of every peer GPU (read over NVLink); `id_scale / id_add` turn a local row into a vid (row * W + rank).
struct KnnMergeParams {
  PeerTable cand_s, cand_i;        // per source: fp32 [n_lists, qstride, k] / int64 [n_lists, qstride, k]
  int n_src, n_lists, qstride, k, B;
  int id_scale;                    // out id = cand_i * id_scale + src * id_add   (when >= 0)
  int id_add;
  float* out_s; int64_t* out_i;    // [B, k], best first
};

// One CTA per query: the candidate scores of every list are staged in shared memory once (coalesced over the lists), then k
// selection passes (thread-local scan -> warp shuffle -> cross-warp reduce) pick the best remaining candidate each.
__global__ void __launch_bounds__(256) knn_merge_kernel(const KnnMergeParams p) {
  extern __shared__ float sc[];                 // [total] candidate scores, -FLT_MAX = invalid / already taken
  __shared__ float red_s[8];
  __shared__ int red_c[8];
  const int q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per_src = p.n_lists * p.k;
  const int total = p.n_src * per_src;
  auto offset_of = [&](int c, int& src) -> size_t {
    src = c / per_src;
    const int rem = c - src * per_src;
    const int l = rem / p.k, e = rem - l * p.k;
    return ((size_t)l * p.qstride + q) * p.k + e;
  };
  for (int c = tid; c < total; c += 256) {
    int src;
    const size_t off = offset_of(c, src);
    const float s = reinterpret_cast<const float*>(p.cand_s.p[src])[off];
    const long long id = reinterpret_cast<const int64_t*>(p.cand_i.p[src])[off];
    sc[c] = id < 0 ? -FLT_MAX : s;
  }
  __syncthreads();
  for (int j = 0; j < p.k; ++j) {
    float best = -FLT_MAX;
    int best_c = -1;
    for (int c = tid; c < total; c += 256) {
      const float s = sc[c];
      if (s > best) { best = s; best_c = c; }            // ascending c inside a thread: the lowest position wins ties
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oc = __shfl_xor_sync(0xffffffffu, best_c, o);
      if (oc >= 0 && (best_c < 0 || ob > best || (ob == best && oc < best_c))) { best = ob; best_c = oc; }
    }
    if (lane == 0) { red_s[warp] = best; red_c[warp] = best_c; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 8; ++w)
        if (red_c[w] >= 0 && (best_c < 0 || red_s[w] > best || (red_s[w] == best && red_c[w] < best_c))) { best = red_s[w]; best_c = red_c[w]; }
      if (best_c < 0 || best == -FLT_MAX) { p.out_s[(size_t)q * p.k + j] = -FLT_MAX; p.out_i[(size_t)q * p.k + j] = -1; }
      else {
        int src;
        const size_t off = offset_of(best_c, src);
        const long long id = reinterpret_cast<const int64_t*>(p.cand_i.p[src])[off];
        p.out_s[(size_t)q * p.k + j] = best;
        p.out_i[(size_t)q * p.k + j] = p.id_scale > 0 ? id * p.id_scale + (long long)src * p.id_add : id;
        sc[best_c] = -FLT_MAX;                               // taken
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// IVF-flat list scan: one CTA per (query, probed list).  The work per pair is tiny (a few thousand rows x d) and every
// query probes different lists, so this is a CUDA-core kernel, exact in fp32: half-warps (fp32: whole warps for d > 128)
// stream the list's rows with 16-byte loads, reduce the squared distance / inner product by shuffles, and each warp keeps
// its k best in shared memory behind a threshold.  Output: [nprobe * 4 warps, B, k] candidate lists for knn_merge_kernel.
// ---------------------------------------------------------------------------------------------------------------
struct KnnIvfParams {
  const void* x; int x_dtype; int64_t x_stride; int dim;
  const int64_t* order;        // rows grouped by list
  const int64_t* offsets;      // [nlist + 1]
  const float* q;              // [B, dim] fp32
  const int64_t* probes;       // [B, nprobe]
  int B, nprobe, k, metric;    // metric 0: -|q - x|^2, 1: <q, x>
  float* out_s; int64_t* out_i;   // [nprobe * 4, B, k]
};

constexpr int kIvfWarps = 4;

__global__ void __launch_bounds__(kIvfWarps * 32) knn_ivf_scan_kernel(const KnnIvfParams p) {
  extern __shared__ float ivf_smem[];
  float* sq = ivf_smem;                                   // [dim] the query
  float* tv = sq + ((p.dim + 3) & ~3);                    // [warps][k] kept scores
  int* ti = reinterpret_cast<int*>(tv + kIvfWarps * p.k); // [warps][k] kept positions inside the list
  const int probe = blockIdx.x, qi = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int f = tid; f < p.dim; f += blockDim.x) sq[f] = p.q[(size_t)qi * p.dim + f];
  for (int e = tid; e < kIvfWarps * p.k; e += blockDim.x) { tv[e] = -FLT_MAX; ti[e] = -1; }
  __syncthreads();
  const int64_t l = p.probes[(size_t)qi * p.nprobe + probe];
  const int64_t lo = p.offsets[l], hi = p.offsets[l + 1];
  const int vec = p.x_dtype == 0 ? 4 : 8;                  // elements per 16-byte chunk
  const int chunks = (p.dim + vec - 1) / vec;
  // lanes per row: the smallest power of two >= chunks (<= 32); wider rows loop over chunk groups
  int lpr = 1;
  while (lpr < chunks && lpr < 32) lpr <<= 1;
  const int rows_per_iter = 32 / lpr;
  const int sub = lane / lpr, lig = lane % lpr;
  float* mv = tv + warp * p.k;
  int* mi = ti + warp * p.k;
  float thr = -FLT_MAX;
  int thr_pos = 0;
  for (int64_t base = lo + (int64_t)warp * rows_per_iter; base < hi; base += (int64_t)kIvfWarps * rows_per_iter) {
    const int64_t pos = base + sub;
    float acc = 0.f;
    if (pos < hi) {
      const int64_t row = __ldg(p.order + pos);
      for (int c = lig; c < chunks; c += lpr) {
        float xv[8];
        const int f0 = c * vec;
        if (p.x_dtype == 0) {
          const float4 t = ld_nc_f4(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.x) + row * p.x_stride) + c);
          xv[0] = t.x; xv[1] = t.y; xv[2] = t.z; xv[3] = t.w;
        } else {
          const uint4 t = ld_nc_u4(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.x) + row * p.x_stride) + c);
          float2 a;
          a = unpack_bf16x2(t.x); xv[0] = a.x; xv[1] = a.y; a = unpack_bf16x2(t.y); xv[2] = a.x; xv[3] = a.y;
          a = unpack_bf16x2(t.z); xv[4] = a.x; xv[5] = a.y; a = unpack_bf16x2(t.w); xv[6] = a.x; xv[7] = a.y;
        }
        for (int i = 0; i < vec; ++i) {
          if (f0 + i < p.dim) {
            const float qv = sq[f0 + i];
            if (p.metric == 1) acc = fmaf(qv, xv[i], acc);
            else { const float dlt = qv - xv[i]; acc = fmaf(-dlt, dlt, acc); }
          }
        }
      }
    }
    for (int o = lpr >> 1; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    // the group leaders hold the scores of this iteration's rows: lane 0 folds them into the warp's list
    for (int g = 0; g < rows_per_iter; ++g) {
      const float sc = __shfl_sync(0xffffffffu, acc, g * lpr);
      const int64_t pg = base + g;
      if (pg < hi && sc > thr) {                            // warp-uniform branch
        if (lane == 0) { mv[thr_pos] = sc; mi[thr_pos] = (int)(pg - lo); }
        __syncwarp();
        float m = FLT_MAX; int mp = 0;                      // new threshold = smallest kept score
        for (int e = lane; e < p.k; e += 32) { const float v = mv[e]; if (v < m) { m = v; mp = e; } }
        for (int o = 16; o > 0; o >>= 1) {
          const float om = __shfl_xor_sync(0xffffffffu, m, o);
          const int op = __shfl_xor_sync(0xffffffffu, mp, o);
          if (om < m || (om == m && op < mp)) { m = om; mp = op; }
        }
        thr = m; thr_pos = mp;
      }
    }
  }
  __syncwarp();
  const size_t ob = (((size_t)probe * kIvfWarps + warp) * p.B + qi) * p.k;
  for (int e = lane; e < p.k; e += 32) {
    const int pi = mi[e];
    p.out_s[ob + e] = mv[e];
    p.out_i[ob + e] = pi >= 0 ? __ldg(p.order + lo + pi) : -1;
  }
}

static void launch_merge(const KnnMergeParams& m, cudaStream_t stream) {
  const size_t smem = (size_t)m.n_src * m.n_lists * m.k * sizeof(float);
  TORCH_CHECK(smem <= 200 * 1024, "too many candidates for the merge kernel's shared-memory stage");
  static bool attr_done = false;
  if (!attr_done) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(knn_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr_done = true;
  }
  knn_merge_kernel<<<(unsigned)m.B, 256, smem, stream>>>(m);
}

// scores / rows of the k best database rows for up to 128 queries.  x: local [n, stride] fp32|bf16; q: bf16 [128, dpad].
// Returns (scores [B, k] best first, rows [B, k]) - rows index x (or row_list's values).
std::vector<at::Tensor> knn_flat_topk(const at::Tensor& x, int64_t dim, const c10::optional<at::Tensor>& x_norm,
                                      const c10::optional<at::Tensor>& row_list, const at::Tensor& q, int64_t B, int64_t k) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && (x.scalar_type() == at::kFloat || x.scalar_type() == at::kBFloat16));
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kBFloat16 && q.dim() == 2 && q.size(0) == kKnnQ && q.is_contiguous() &&
              q.size(1) % 64 == 0 && q.size(1) >= dim && q.size(1) <= 512, "q must be bf16 [128, dpad] (dpad multiple of 64, <= 512)");
  TORCH_CHECK(k >= 1 && k <= kKnnMaxK && B >= 1 && B <= kKnnQ);
  TORCH_CHECK(x.scalar_type() == at::kFloat || (x.stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0),
              "bf16 tables need 16-byte aligned rows");
  c10::cuda::CUDAGuard guard(x.device());
  KnnParams p;
  std::memset(&p, 0, sizeof(p));
  p.x = x.data_ptr(); p.x_dtype = x.scalar_type() == at::kFloat ? 0 : 1; p.x_stride = x.stride(0);
  p.dim = (int)dim; p.dpad = (int)q.size(1); p.k = (int)k; p.B = (int)B;
  p.q = reinterpret_cast<const __nv_bfloat16*>(q.data_ptr());
  at::Tensor nrm, rl;
  if (x_norm.has_value() && x_norm->defined()) { nrm = x_norm->contiguous(); TORCH_CHECK(nrm.scalar_type() == at::kFloat && nrm.numel() >= x.size(0)); p.x_norm = nrm.data_ptr<float>(); }
  p.n = x.size(0);
  if (row_list.has_value() && row_list->defined()) { rl = row_list->contiguous(); check_cuda_i64(rl, "row_list"); p.row_list = rl.data_ptr<int64_t>(); p.n = rl.numel(); }
  auto of = x.options().dtype(at::kFloat);
  auto oi = x.options().dtype(at::kLong);
  auto out_s = at::empty({B, k}, of);
  auto out_i = at::empty({B, k}, oi);
  if (p.n == 0) { out_s.fill_(-FLT_MAX); out_i.fill_(-1); return {out_s, out_i}; }
  const int sms = sm_count();
  int64_t slabs = (p.n + kKnnSlab - 1) / kKnnSlab;
  int grid = (int)std::min<int64_t>(sms, slabs);
  p.rows_per_cta = (slabs + grid - 1) / grid * kKnnSlab;
  grid = (int)((p.n + p.rows_per_cta - 1) / p.rows_per_cta);
  auto part_s = at::empty({grid, kKnnQ, k}, of);
  auto part_i = at::empty({grid, kKnnQ, k}, oi);
  p.out_s = part_s.data_ptr<float>(); p.out_i = part_i.data_ptr<int64_t>();
  const size_t tile = (size_t)(p.dpad / 64) * 128 * 128;
  auto smem_for = [&](int nbuf) {
    return 1024 + (size_t)(1 + nbuf) * tile + (size_t)nbuf * kKnnSlab * 4 + (size_t)kKnnQ * kKnnScoreLd * 4 + (size_t)k * kKnnQ * 8 + 4 * 8;
  };
  p.n_xbuf = smem_for(2) <= 232448 ? 2 : 1;                  // wide queries / large k: one slab buffer, no load-MMA overlap
  const size_t smem = smem_for(p.n_xbuf);
  TORCH_CHECK(smem <= 232448, "query width too large for the fused KNN tile");
  static size_t attr = 0;
  if (smem > attr) { C10_CUDA_CHECK(cudaFuncSetAttribute(knn_flat_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  auto stream = at::cuda::getCurrentCUDAStream();
  knn_flat_kernel<<<grid, kKnnThreads, smem, stream>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  KnnMergeParams m;
  std::memset(&m, 0, sizeof(m));
  m.cand_s.p[0] = part_s.data_ptr(); m.cand_i.p[0] = part_i.data_ptr();
  m.n_src = 1; m.n_lists = grid; m.qstride = kKnnQ; m.k = (int)k; m.B = (int)B; m.id_scale = 0;
  m.out_s = out_s.data_ptr<float>(); m.out_i = out_i.data_ptr<int64_t>();
  launch_merge(m, stream);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {out_s, out_i};
}

// cross-GPU merge: every rank holds its local (scores [B, k], rows [B, k]) in a SYMMETRIC buffer; each rank reads all
// peers' lists over NVLink and keeps the global k best as vids (row * world + rank).  ptrs: CPU int64 [2, world].
std::vector<at::Tensor> knn_merge_peers(const at::Tensor& ptrs, int64_t world, int64_t B, int64_t k, const at::Tensor& like) {
  TORCH_CHECK(ptrs.device().is_cpu() && ptrs.scalar_type() == at::kLong && ptrs.numel() == 2 * world && world <= kMaxWorld);
  c10::cuda::CUDAGuard guard(like.device());
  KnnMergeParams m;
  std::memset(&m, 0, sizeof(m));
  const int64_t* d = ptrs.data_ptr<int64_t>();
  for (int r = 0; r < world; ++r) { m.cand_s.p[r] = reinterpret_cast<const void*>(d[r]); m.cand_i.p[r] = reinterpret_cast<const void*>(d[world + r]); }
  m.n_src = (int)world; m.n_lists = 1; m.qstride = (int)B; m.k = (int)k; m.B = (int)B; m.id_scale = (int)world; m.id_add = 1;
  auto out_s = at::empty({B, k}, like.options().dtype(at::kFloat));
  auto out_i = at::empty({B, k}, like.options().dtype(at::kLong));
  m.out_s = out_s.data_ptr<float>(); m.out_i = out_i.data_ptr<int64_t>();
  launch_merge(m, at::cuda::getCurrentCUDAStream());
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {out_s, out_i};
}

// IVF-flat search: (scores [B, k] best first, rows [B, k]) over the probed lists of every query, exact in fp32.
std::vector<at::Tensor> knn_ivf_search(const at::Tensor& x, int64_t dim, const at::Tensor& order, const at::Tensor& offsets, const at::Tensor& q,
                                       const at::Tensor& probes, int64_t k, int64_t metric) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.stride(1) == 1 && (x.scalar_type() == at::kFloat || x.scalar_type() == at::kBFloat16));
  TORCH_CHECK((x.stride(0) * x.element_size()) % 16 == 0 && (reinterpret_cast<uintptr_t>(x.data_ptr()) & 15) == 0, "rows must be 16-byte aligned");
  check_cuda_i64(order, "order"); check_cuda_i64(offsets, "offsets"); check_cuda_i64(probes, "probes");
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kFloat && q.dim() == 2 && q.size(1) == dim && q.is_contiguous());
  TORCH_CHECK(probes.dim() == 2 && probes.size(0) == q.size(0) && probes.is_contiguous() && order.is_contiguous() && offsets.is_contiguous());
  TORCH_CHECK(k >= 1 && k <= kKnnMaxK);
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t B = q.size(0), nprobe = probes.size(1);
  auto of = x.options().dtype(at::kFloat);
  auto oi = x.options().dtype(at::kLong);
  auto out_s = at::empty({B, k}, of);
  auto out_i = at::empty({B, k}, oi);
  if (B == 0) return {out_s, out_i};
  auto part_s = at::empty({nprobe * kIvfWarps, B, k}, of);
  auto part_i = at::empty({nprobe * kIvfWarps, B, k}, oi);
  KnnIvfParams p;
  p.x = x.data_ptr(); p.x_dtype = x.scalar_type() == at::kFloat ? 0 : 1; p.x_stride = x.stride(0); p.dim = (int)dim;
  p.order = order.data_ptr<int64_t>(); p.offsets = offsets.data_ptr<int64_t>(); p.q = q.data_ptr<float>();
  p.probes = probes.data_ptr<int64_t>(); p.B = (int)B; p.nprobe = (int)nprobe; p.k = (int)k; p.metric = (int)metric;
  p.out_s = part_s.data_ptr<float>(); p.out_i = part_i.data_ptr<int64_t>();
  auto stream = at::cuda::getCurrentCUDAStream();
  const size_t smem = (((size_t)dim + 3) & ~(size_t)3) * 4 + (size_t)kIvfWarps * k * 8;
  knn_ivf_scan_kernel<<<dim3((unsigned)nprobe, (unsigned)B), kIvfWarps * 32, smem, stream>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  KnnMergeParams m;
  std::memset(&m, 0, sizeof(m));
  m.cand_s.p[0] = part_s.data_ptr(); m.cand_i.p[0] = part_i.data_ptr();
  m.n_src = 1; m.n_lists = (int)(nprobe * kIvfWarps); m.qstride = (int)B; m.k = (int)k; m.B = (int)B; m.id_scale = 0;
  m.out_s = out_s.data_ptr<float>(); m.out_i = out_i.data_ptr<int64_t>();
  launch_merge(m, stream);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {out_s, out_i};
}

// ---------------------------------------------------------------------------------------------------------------
// IVF-PQ list scan (index_factory.cc:40-50 'ivfpq'): one CTA per (query, probed list).  Rows are stored as M one-byte
// codes of their residual to the list centroid; the CTA first builds the asymmetric-distance table
// LUT[m][c] = -|r_m - codebook[m][c]|^2 (L2, r = q - centroid) or <q_m, codebook[m][c]> (inner product, plus the constant
// <q, centroid>) in shared memory, then every lane scores one row per iteration with M shared-memory look-ups and the
// warps keep their k best behind a threshold exactly like the IVF-flat scan.  Output: [nprobe * 8 warps, B, k].
// ---------------------------------------------------------------------------------------------------------------
struct KnnPqParams {
  const uint8_t* codes;        // [n, M] in list order (position-indexed)
  const int64_t* order;        // position -> row
  const int64_t* offsets;      // [nlist + 1]
  const float* q;              // [B, dim]  (dim = M * dsub, zero padded)
  const int64_t* probes;       // [B, nprobe]
  const float* centroids;      // [nlist, dim]
  const float* codebooks;      // [M, 256, dsub]
  int B, nprobe, k, metric, M, dsub;
  float* out_s; int64_t* out_i;   // [nprobe * 8, B, k]
};

constexpr int kPqWarps = 8;

__global__ void __launch_bounds__(kPqWarps * 32) knn_ivfpq_scan_kernel(const KnnPqParams p) {
  extern __shared__ float pq_smem[];
  const int dim = p.M * p.dsub;
  float* lut = pq_smem;                                   // [M][256]
  float* sr = lut + p.M * 256;                            // [dim] residual (L2) or the query (inner product)
  float* tv = sr + ((dim + 3) & ~3);                      // [warps][k]
  int* ti = reinterpret_cast<int*>(tv + kPqWarps * p.k);  // [warps][k]
  __shared__ float s_bias;
  const int probe = blockIdx.x, qi = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int64_t l = p.probes[(size_t)qi * p.nprobe + probe];
  const int64_t lo = p.offsets[l], hi = p.offsets[l + 1];
  const float* cen = p.centroids + (size_t)l * dim;
  for (int f = tid; f < dim; f += blockDim.x) {
    const float qv = p.q[(size_t)qi * dim + f];
    sr[f] = p.metric == 1 ? qv : qv - __ldg(cen + f);
  }
  for (int e = tid; e < kPqWarps * p.k; e += blockDim.x) { tv[e] = -FLT_MAX; ti[e] = -1; }
  if (warp == 0) {                                         // <q, centroid>: the part of an inner product the codes do not carry
    float b = 0.f;
    if (p.metric == 1) for (int f = lane; f < dim; f += 32) b = fmaf(p.q[(size_t)qi * dim + f], __ldg(cen + f), b);
    for (int o = 16; o > 0; o >>= 1) b += __shfl_xor_sync(0xffffffffu, b, o);
    if (lane == 0) s_bias = b;
  }
  __syncthreads();
  if (hi > lo) {
    for (int e = tid; e < p.M * 256; e += blockDim.x) {
      const int m = e >> 8;
      const float* cb = p.codebooks + (size_t)e * p.dsub;
      const float* r = sr + m * p.dsub;
      float acc = 0.f;
      for (int d = 0; d < p.dsub; ++d) {
        const float c = __ldg(cb + d);
        if (p.metric == 1) acc = fmaf(r[d], c, acc);
        else { const float dlt = r[d] - c; acc = fmaf(-dlt, dlt, acc); }
      }
      lut[e] = acc;
    }
  }
  __syncthreads();
  const float bias = s_bias;
  float* mv = tv + warp * p.k;
  int* mi = ti + warp * p.k;
  float thr = -FLT_MAX;
  int thr_pos = 0;
  const bool words = (p.M & 3) == 0;
  for (int64_t base = lo + (int64_t)warp * 32; base < hi; base += (int64_t)kPqWarps * 32) {
    const int64_t pos = base + lane;
    float acc = bias;
    if (pos < hi) {
      const uint8_t* code = p.codes + (size_t)pos * p.M;
      if (words) {
        const uint32_t* cw = reinterpret_cast<const uint32_t*>(code);
        for (int m = 0; m < p.M; m += 4) {
          const uint32_t w = __ldg(cw + (m >> 2));
          acc += lut[(m + 0) * 256 + (w & 255u)];
          acc += lut[(m + 1) * 256 + ((w >> 8) & 255u)];
          acc += lut[(m + 2) * 256 + ((w >> 16) & 255u)];
          acc += lut[(m + 3) * 256 + (w >> 24)];
        }
      } else {
        for (int m = 0; m < p.M; ++m) acc += lut[m * 256 + __ldg(code + m)];
      }
    }
    unsigned cand = __ballot_sync(0xffffffffu, pos < hi && acc > thr);
    while (cand) {                                          // warp-uniform: lanes whose score beats the threshold
      const int g = __ffs(cand) - 1;
      cand &= cand - 1;
      const float sc = __shfl_sync(0xffffffffu, acc, g);
      if (sc > thr) {
        if (lane == 0) { mv[thr_pos] = sc; mi[thr_pos] = (int)(base + g - lo); }
        __syncwarp();
        float mn = FLT_MAX; int mp = 0;
        for (int e = lane; e < p.k; e += 32) { const float v = mv[e]; if (v < mn) { mn = v; mp = e; } }
        for (int o = 16; o > 0; o >>= 1) {
          const float om = __shfl_xor_sync(0xffffffffu, mn, o);
          const int op = __shfl_xor_sync(0xffffffffu, mp, o);
          if (om < mn || (om == mn && op < mp)) { mn = om; mp = op; }
        }
        thr = mn; thr_pos = mp;
        __syncwarp();
      }
    }
  }
  __syncwarp();
  const size_t ob = (((size_t)probe * kPqWarps + warp) * p.B + qi) * p.k;
  for (int e = lane; e < p.k; e += 32) {
    const int pi = mi[e];
    p.out_s[ob + e] = mv[e];
    p.out_i[ob + e] = pi >= 0 ? __ldg(p.order + lo + pi) : -1;
  }
}

// IVF-PQ search: (approximate scores [B, k] best first, rows [B, k]) over the probed lists of every query.
std::vector<at::Tensor> knn_ivfpq_search(const at::Tensor& codes, const at::Tensor& order, const at::Tensor& offsets, const at::Tensor& q,
                                         const at::Tensor& probes, const at::Tensor& centroids, const at::Tensor& codebooks, int64_t k,
                                         int64_t metric) {
  TORCH_CHECK(codes.is_cuda() && codes.scalar_type() == at::kByte && codes.dim() == 2 && codes.is_contiguous(), "codes must be uint8 [n, M]");
  TORCH_CHECK(codebooks.is_cuda() && codebooks.scalar_type() == at::kFloat && codebooks.dim() == 3 && codebooks.size(1) == 256 &&
              codebooks.is_contiguous() && codebooks.size(0) == codes.size(1), "codebooks must be fp32 [M, 256, dsub]");
  const int64_t M = codes.size(1), dsub = codebooks.size(2), dim = M * dsub;
  check_cuda_i64(order, "order"); check_cuda_i64(offsets, "offsets"); check_cuda_i64(probes, "probes");
  TORCH_CHECK(q.is_cuda() && q.scalar_type() == at::kFloat && q.dim() == 2 && q.size(1) == dim && q.is_contiguous(), "q must be fp32 [B, M * dsub]");
  TORCH_CHECK(centroids.is_cuda() && centroids.scalar_type() == at::kFloat && centroids.dim() == 2 && centroids.size(1) == dim &&
              centroids.is_contiguous() && centroids.size(0) + 1 == offsets.numel());
  TORCH_CHECK(probes.dim() == 2 && probes.size(0) == q.size(0) && probes.is_contiguous() && order.is_contiguous() && offsets.is_contiguous());
  TORCH_CHECK(order.numel() == codes.size(0));
  TORCH_CHECK(k >= 1 && k <= kKnnMaxK && M >= 1 && M <= 128);
  TORCH_CHECK((reinterpret_cast<uintptr_t>(codes.data_ptr()) & 3) == 0);
  c10::cuda::CUDAGuard guard(codes.device());
  const int64_t B = q.size(0), nprobe = probes.size(1);
  auto of = q.options().dtype(at::kFloat);
  auto oi = q.options().dtype(at::kLong);
  auto out_s = at::empty({B, k}, of);
  auto out_i = at::empty({B, k}, oi);
  if (B == 0) return {out_s, out_i};
  auto part_s = at::empty({nprobe * kPqWarps, B, k}, of);
  auto part_i = at::empty({nprobe * kPqWarps, B, k}, oi);
  KnnPqParams p;
  p.codes = codes.data_ptr<uint8_t>(); p.order = order.data_ptr<int64_t>(); p.offsets = offsets.data_ptr<int64_t>();
  p.q = q.data_ptr<float>(); p.probes = probes.data_ptr<int64_t>(); p.centroids = centroids.data_ptr<float>();
  p.codebooks = codebooks.data_ptr<float>();
  p.B = (int)B; p.nprobe = (int)nprobe; p.k = (int)k; p.metric = (int)metric; p.M = (int)M; p.dsub = (int)dsub;
  p.out_s = part_s.data_ptr<float>(); p.out_i = part_i.data_ptr<int64_t>();
  auto stream = at::cuda::getCurrentCUDAStream();
  const size_t smem = (size_t)M * 256 * 4 + (((size_t)dim + 3) & ~(size_t)3) * 4 + (size_t)kPqWarps * k * 8;
  TORCH_CHECK(smem <= 200 * 1024, "PQ look-up table too large for shared memory");
  static size_t attr = 48 * 1024;
  if (smem > attr) { C10_CUDA_CHECK(cudaFuncSetAttribute(knn_ivfpq_scan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); attr = smem; }
  knn_ivfpq_scan_kernel<<<dim3((unsigned)nprobe, (unsigned)B), kPqWarps * 32, smem, stream>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  KnnMergeParams m;
  std::memset(&m, 0, sizeof(m));
  m.cand_s.p[0] = part_s.data_ptr(); m.cand_i.p[0] = part_i.data_ptr();
  m.n_src = 1; m.n_lists = (int)(nprobe * kPqWarps); m.qstride = (int)B; m.k = (int)k; m.B = (int)B; m.id_scale = 0;
  m.out_s = out_s.data_ptr<float>(); m.out_i = out_i.data_ptr<int64_t>();
  launch_merge(m, stream);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {out_s, out_i};
}

}  // namespace glb
