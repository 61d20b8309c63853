// Batch normalisation of the hidden layers of the fused GraphSAGE trainer (engine/fast_sage.py, EgoGraphSAGE with
// batch_norm=True).  A hidden layer's launch writes Z_l (fp32, no bias, no ReLU) for all of its segments (hop tensors);
// each segment s is normalised with its own batch statistics, as the reference's EgoGNN calls bn_func once per hop
// tensor:
//
//   H = dropout(relu(gamma (Z - mu_s) rstd_s + beta)),   rstd_s = 1 / sqrt(var_s + eps), var_s biased
//
// Four memory-bound kernels over the layer's [rows, C] buffers, all per-segment column statistics in fp32:
//   bn_colsum_kernel<false>   forward statistics: per segment and column the sums of d = z - K and d^2, K = the column's
//                             value in the segment's first row (shifted sums: the variance keeps its precision when
//                             |mean| >> std, where E[z^2] - E[z]^2 would cancel).  CTAs of 256-row chunks write
//                             partial sums; the last CTA of a column block (atomic ticket) adds them up in chunk order
//                             (deterministic), writes mean / rstd and updates the BatchNorm1d module's running_mean /
//                             running_var (unbiased) once per segment in hop order, and num_batches_tracked += nseg
//   bn_apply_kernel           H = dropout(relu(BN(Z))) as bf16, the mask drawn by dropout_philox (dropout.cuh) at
//                             (row of the layer's buffer, column) - the forward epilogue's mask, bit for bit
//   bn_colsum_kernel<true>    backward: per segment and column sum(dY) and sum(dY x^), x^ recomputed from Z, mu, rstd;
//                             the finalising CTA adds their sums over the segments to d(beta) and d(gamma)
//   bn_bwd_apply_kernel       dZ = gamma rstd (dY - sum(dY) / n - x^ sum(dY x^) / n) as bf16
// dY (the gradient of the BN output, ReLU and dropout routed) comes from sage_bwd_dz_kernel, sage_bwd_dw's dZ-only mode.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cmath>
#include <cstring>
#include "host_utils.h"
#include "dropout.cuh"

namespace glb {

constexpr int kBnMaxSegs = 4;
constexpr int kBnThreads = 256;
constexpr int kBnCols = 64;                         // columns per CTA of the column sums: 16 lanes x 4 columns
constexpr int kBnLanes = kBnThreads / (kBnCols / 4); // 16 row lanes
constexpr int kBnChunk = 256;                       // rows per CTA of the column sums: 16 per lane, all loads in flight

struct BnSegs {
  int row0[kBnMaxSegs + 1];                         // segment s = rows [row0[s], row0[s + 1])
  int chunk0[kBnMaxSegs + 1];                       // its kBnChunk-row chunks are [chunk0[s], chunk0[s + 1])
  int nseg;
};

__device__ __forceinline__ int bn_seg_of_row(const BnSegs& g, int r) {
  int s = 0;
#pragma unroll
  for (int i = 1; i < kBnMaxSegs; ++i)
    if (i < g.nseg && r >= g.row0[i]) s = i;
  return s;
}

struct BnSumParams {
  BnSegs g;
  const float* z; int ldz;
  const __nv_bfloat16* dy; int lddy;               // backward only
  int C;
  float* part;                                     // [chunks][2][C] partial sums
  int* ticket;                                     // [column blocks], zero between launches
  float* mean; float* rstd;                        // [nseg][C]: written (forward) or read (backward)
  // forward: the BatchNorm1d buffers
  float* run_mean; float* run_var; long long* nbt;
  float eps, momentum;
  // backward: per segment sum(dY) and sum(dY x^) [nseg][2][C], and the parameters' gradients (accumulated)
  float* gsum; float* dgamma; float* dbeta;
};

template <bool BWD>
__global__ void __launch_bounds__(kBnThreads) bn_colsum_kernel(const __grid_constant__ BnSumParams p) {
  __shared__ float sred[2][kBnLanes][kBnCols];
  __shared__ float sfin[2][4][kBnCols];
  __shared__ int s_last;
  const int tid = threadIdx.x, lane_c = tid & 15, lane_r = tid >> 4;
  const int chunk = blockIdx.y;
  int s = 0;
#pragma unroll
  for (int i = 1; i < kBnMaxSegs; ++i)
    if (i < p.g.nseg && chunk >= p.g.chunk0[i]) s = i;
  const int seg_r0 = p.g.row0[s], seg_r1 = p.g.row0[s + 1];
  const int r_begin = seg_r0 + (chunk - p.g.chunk0[s]) * kBnChunk;
  const int r_end = min(seg_r1, r_begin + kBnChunk);
  const int c = blockIdx.x * kBnCols + lane_c * 4;
  const bool col_ok = c < p.C;
  float a0[4] = {0.f, 0.f, 0.f, 0.f}, a1[4] = {0.f, 0.f, 0.f, 0.f};
  if (col_ok) {
    float k[4], sc[4];
    if constexpr (BWD) {
      const float4 m = *reinterpret_cast<const float4*>(p.mean + (size_t)s * p.C + c);
      const float4 rs = *reinterpret_cast<const float4*>(p.rstd + (size_t)s * p.C + c);
      k[0] = m.x; k[1] = m.y; k[2] = m.z; k[3] = m.w; sc[0] = rs.x; sc[1] = rs.y; sc[2] = rs.z; sc[3] = rs.w;
    } else {
      const float4 m = *reinterpret_cast<const float4*>(p.z + (size_t)seg_r0 * p.ldz + c);
      k[0] = m.x; k[1] = m.y; k[2] = m.z; k[3] = m.w;
    }
#pragma unroll
    for (int i = 0; i < kBnChunk / kBnLanes; ++i) {
      const int r = r_begin + lane_r + i * kBnLanes;
      const bool in = r < r_end;               // rows past the chunk add zeros (d = 0 - 0, dY = 0)
      const float4 zv = in ? *reinterpret_cast<const float4*>(p.z + (size_t)r * p.ldz + c) : make_float4(k[0], k[1], k[2], k[3]);
      const float zz[4] = {zv.x, zv.y, zv.z, zv.w};
      if constexpr (BWD) {
        const uint2 u = in ? *reinterpret_cast<const uint2*>(p.dy + (size_t)r * p.lddy + c) : make_uint2(0u, 0u);
        const float2 d01 = unpack_bf16x2(u.x), d23 = unpack_bf16x2(u.y);
        const float dd[4] = {d01.x, d01.y, d23.x, d23.y};
#pragma unroll
        for (int j = 0; j < 4; ++j) { a0[j] += dd[j]; a1[j] = fmaf(dd[j], (zz[j] - k[j]) * sc[j], a1[j]); }
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) { const float d = zz[j] - k[j]; a0[j] += d; a1[j] = fmaf(d, d, a1[j]); }
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) { sred[0][lane_r][lane_c * 4 + j] = a0[j]; sred[1][lane_r][lane_c * 4 + j] = a1[j]; }
  __syncthreads();
  if (tid < 2 * kBnCols) {
    const int w = tid / kBnCols, cc = tid % kBnCols, col = blockIdx.x * kBnCols + cc;
    float v = 0.f;
#pragma unroll
    for (int i = 0; i < kBnLanes; ++i) v += sred[w][i][cc];
    if (col < p.C) p.part[((size_t)chunk * 2 + w) * p.C + col] = v;
  }
  // the last CTA of this column block finalises every segment
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(p.ticket + blockIdx.x, 1) == (int)gridDim.y - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const int cc = tid % kBnCols, q = tid / kBnCols, col = blockIdx.x * kBnCols + cc;
  float dg = 0.f, db = 0.f;
  for (int sg = 0; sg < p.g.nseg; ++sg) {
    // four threads per column sum every fourth chunk of the segment; thread q = 0 adds the four in order
    float v0 = 0.f, v1 = 0.f;
    if (col < p.C)
#pragma unroll 4
      for (int ch = p.g.chunk0[sg] + q; ch < p.g.chunk0[sg + 1]; ch += 4) {
        v0 += __ldcg(p.part + ((size_t)ch * 2) * p.C + col);
        v1 += __ldcg(p.part + ((size_t)ch * 2 + 1) * p.C + col);
      }
    sfin[0][q][cc] = v0; sfin[1][q][cc] = v1;
    __syncthreads();
    if (q == 0 && col < p.C) {
      const float s0 = ((sfin[0][0][cc] + sfin[0][1][cc]) + sfin[0][2][cc]) + sfin[0][3][cc];
      const float s1 = ((sfin[1][0][cc] + sfin[1][1][cc]) + sfin[1][2][cc]) + sfin[1][3][cc];
      const float n = (float)(p.g.row0[sg + 1] - p.g.row0[sg]);
      if constexpr (BWD) {
        p.gsum[((size_t)sg * 2) * p.C + col] = s0;
        p.gsum[((size_t)sg * 2 + 1) * p.C + col] = s1;
        db += s0; dg += s1;
      } else {
        const float md = s0 / n;
        const float var = fmaxf(s1 / n - md * md, 0.f);
        const float mu = __ldcg(p.z + (size_t)p.g.row0[sg] * p.ldz + col) + md;
        p.mean[(size_t)sg * p.C + col] = mu;
        p.rstd[(size_t)sg * p.C + col] = rsqrtf(var + p.eps);
        const float m = p.momentum;
        p.run_mean[col] = (1.f - m) * p.run_mean[col] + m * mu;
        p.run_var[col] = (1.f - m) * p.run_var[col] + m * (var * n / (n - 1.f));
      }
    }
    __syncthreads();
  }
  if constexpr (BWD) {
    if (q == 0 && col < p.C) { p.dbeta[col] += db; p.dgamma[col] += dg; }
  } else {
    if (blockIdx.x == 0 && tid == 0) *p.nbt += p.g.nseg;
  }
  if (tid == 0) p.ticket[blockIdx.x] = 0;
}

// H = dropout(relu(gamma (Z - mu) rstd + beta)) -> bf16.  Thread (row, 32-column group g, q < 4) holds the eight columns
// 32 g + 8 w + 2 q + e (w < 4, e < 2) that one dropout_philox call covers.
struct BnApplyParams {
  BnSegs g;
  const float* z; int ldz;
  const float* mean; const float* rstd;
  const float* gamma; const float* beta;
  __nv_bfloat16* h; int ldh;
  int rows, C, groups;                            // groups = 4 * ceil(C / 32) threads per row
  const unsigned long long* drop_state;           // or null (no dropout)
  uint32_t drop_thr, drop_layer;
  float drop_scale;
};

__global__ void __launch_bounds__(kBnThreads) bn_apply_kernel(const __grid_constant__ BnApplyParams p) {
  const long long t = (long long)blockIdx.x * kBnThreads + threadIdx.x;
  if (t >= (long long)p.rows * p.groups) return;
  const int r = (int)(t / p.groups), gq = (int)(t % p.groups);
  const int c0 = (gq >> 2) * 32 + 2 * (gq & 3);
  const int s = bn_seg_of_row(p.g, r);
  uint4 u = make_uint4(0u, 0u, 0u, 0u);
  if (p.drop_state) u = dropout_philox(p.drop_state, p.drop_layer, (uint32_t)r, (uint32_t)c0);
#pragma unroll
  for (int w = 0; w < 4; ++w) {
    const int c = c0 + 8 * w;
    if (c >= p.C) continue;
    const float2 zv = *reinterpret_cast<const float2*>(p.z + (size_t)r * p.ldz + c);
    const float2 mu = *reinterpret_cast<const float2*>(p.mean + (size_t)s * p.C + c);
    const float2 rs = *reinterpret_cast<const float2*>(p.rstd + (size_t)s * p.C + c);
    const float2 ga = *reinterpret_cast<const float2*>(p.gamma + c);
    const float2 be = *reinterpret_cast<const float2*>(p.beta + c);
    float x0 = fmaxf(fmaf(ga.x, (zv.x - mu.x) * rs.x, be.x), 0.f);
    float x1 = fmaxf(fmaf(ga.y, (zv.y - mu.y) * rs.y, be.y), 0.f);
    if (p.drop_state) {
      const uint32_t bits = w == 0 ? u.x : w == 1 ? u.y : w == 2 ? u.z : u.w;
      x0 = (bits & 0xFFFFu) >= p.drop_thr ? x0 * p.drop_scale : 0.f;
      x1 = (bits >> 16) >= p.drop_thr ? x1 * p.drop_scale : 0.f;
    }
    *reinterpret_cast<uint32_t*>(p.h + (size_t)r * p.ldh + c) = pack_bf16x2(x0, x1);
  }
}

// dZ = gamma rstd (dY - sum(dY) / n - x^ sum(dY x^) / n) -> bf16, eight columns per thread
struct BnBwdParams {
  BnSegs g;
  const float* z; int ldz;
  const __nv_bfloat16* dy; int lddy;
  const float* mean; const float* rstd; const float* gamma; const float* gsum;
  __nv_bfloat16* dz; int lddz;
  int rows, C;
};

__global__ void __launch_bounds__(kBnThreads) bn_bwd_apply_kernel(const __grid_constant__ BnBwdParams p) {
  const int per_row = p.C / 8;
  const long long t = (long long)blockIdx.x * kBnThreads + threadIdx.x;
  if (t >= (long long)p.rows * per_row) return;
  const int r = (int)(t / per_row), c = (int)(t % per_row) * 8;
  const int s = bn_seg_of_row(p.g, r);
  const float inv_n = 1.f / (float)(p.g.row0[s + 1] - p.g.row0[s]);
  const uint4 du = *reinterpret_cast<const uint4*>(p.dy + (size_t)r * p.lddy + c);
  const uint32_t dw[4] = {du.x, du.y, du.z, du.w};
  const float* zr = p.z + (size_t)r * p.ldz + c;
  const float4 za = *reinterpret_cast<const float4*>(zr), zb = *reinterpret_cast<const float4*>(zr + 4);
  const float zz[8] = {za.x, za.y, za.z, za.w, zb.x, zb.y, zb.z, zb.w};
  // the eight columns' statistics and parameters as float4 pairs (C is a multiple of 8, the rows 16-byte aligned)
  float mu[8], rs[8], ga[8], s0[8], s1[8];
  auto ld8 = [&](const float* src, float (&dst)[8]) {
    const float4 a = *reinterpret_cast<const float4*>(src), b = *reinterpret_cast<const float4*>(src + 4);
    dst[0] = a.x; dst[1] = a.y; dst[2] = a.z; dst[3] = a.w; dst[4] = b.x; dst[5] = b.y; dst[6] = b.z; dst[7] = b.w;
  };
  ld8(p.mean + (size_t)s * p.C + c, mu);
  ld8(p.rstd + (size_t)s * p.C + c, rs);
  ld8(p.gamma + c, ga);
  ld8(p.gsum + (size_t)s * 2 * p.C + c, s0);
  ld8(p.gsum + (size_t)s * 2 * p.C + p.C + c, s1);
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 d = unpack_bf16x2(dw[j]);
    float v[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int k = 2 * j + e;
      const float xh = (zz[k] - mu[k]) * rs[k];
      v[e] = ga[k] * rs[k] * ((e ? d.y : d.x) - s0[k] * inv_n - xh * s1[k] * inv_n);
    }
    o[j] = pack_bf16x2(v[0], v[1]);
  }
  *reinterpret_cast<uint4*>(p.dz + (size_t)r * p.lddz + c) = make_uint4(o[0], o[1], o[2], o[3]);
}

// ------------------------------------------------------------------------------------------------ host
static void check_f32(const at::Tensor& t, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.is_contiguous() &&
              (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) == 0, what, " must be a contiguous, 16-byte aligned CUDA fp32 tensor");
}

static void check_rows(const at::Tensor& t, at::ScalarType dt, int rows, int C, const char* what) {
  const int esz = dt == at::kFloat ? 4 : 2;
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == dt && t.dim() == 2 && t.stride(1) == 1 && t.size(0) == rows && t.size(1) >= C &&
              (t.stride(0) * esz) % 16 == 0 && (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15) == 0,
              what, " must be a [rows, >= C] view with 16-byte aligned rows");
}

// offs: the nseg + 1 row offsets of the layer's segments (offs[0] = 0, offs[nseg] = rows); every segment has >= 2 rows
static BnSegs make_segs(const std::vector<int64_t>& offs, int rows) {
  BnSegs g;
  std::memset(&g, 0, sizeof(g));
  const int nseg = (int)offs.size() - 1;
  TORCH_CHECK(nseg >= 1 && nseg <= kBnMaxSegs && offs[0] == 0 && offs[nseg] == rows, "batch norm: 1..", kBnMaxSegs,
              " segments whose offsets cover the rows");
  g.nseg = nseg;
  for (int s = 0; s <= nseg; ++s) {
    g.row0[s] = (int)offs[s];
    if (s < nseg) {
      TORCH_CHECK(offs[s + 1] - offs[s] >= 2, "batch norm needs at least 2 rows per segment");
      g.chunk0[s + 1] = g.chunk0[s] + (int)((offs[s + 1] - offs[s] + kBnChunk - 1) / kBnChunk);
    }
  }
  return g;
}

static void launch_colsum(BnSumParams& p, bool bwd, const at::Tensor& ticket, const at::Tensor& like) {
  const int cblocks = (p.C + kBnCols - 1) / kBnCols;
  TORCH_CHECK(ticket.is_cuda() && ticket.scalar_type() == at::kInt && ticket.numel() >= cblocks,
              "ticket must be a CUDA int32 tensor of >= ceil(C / 64) zeros");
  at::Tensor part = at::empty({(int64_t)p.g.chunk0[p.g.nseg] * 2 * p.C}, like.options().dtype(at::kFloat));
  p.part = part.data_ptr<float>();
  p.ticket = ticket.data_ptr<int>();
  const dim3 grid((unsigned)cblocks, (unsigned)p.g.chunk0[p.g.nseg]);
  if (bwd) bn_colsum_kernel<true><<<grid, kBnThreads, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  else bn_colsum_kernel<false><<<grid, kBnThreads, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// Forward statistics of Z [rows, >= C] fp32: mean / rstd [nseg, C], and the running buffers updated once per segment.
void bn_fwd_stats(const at::Tensor& z, int64_t C, const std::vector<int64_t>& offs, const at::Tensor& ticket,
                  const at::Tensor& mean, const at::Tensor& rstd, const at::Tensor& running_mean, const at::Tensor& running_var,
                  const at::Tensor& num_batches_tracked, double eps, double momentum) {
  TORCH_CHECK(C > 0 && C % 8 == 0, "batch norm width must be a multiple of 8");
  check_rows(z, at::kFloat, (int)z.size(0), (int)C, "z");
  BnSumParams p;
  std::memset(&p, 0, sizeof(p));
  p.g = make_segs(offs, (int)z.size(0));
  p.z = z.data_ptr<float>(); p.ldz = (int)z.stride(0); p.C = (int)C;
  for (const at::Tensor* t : {&mean, &rstd}) { check_f32(*t, "mean / rstd"); TORCH_CHECK(t->numel() >= p.g.nseg * C); }
  for (const at::Tensor* t : {&running_mean, &running_var}) { check_f32(*t, "running_mean / running_var"); TORCH_CHECK(t->numel() == C); }
  TORCH_CHECK(num_batches_tracked.is_cuda() && num_batches_tracked.scalar_type() == at::kLong && num_batches_tracked.numel() == 1);
  TORCH_CHECK(momentum > 0.0 && momentum <= 1.0, "batch norm momentum must be in (0, 1]");
  p.mean = mean.data_ptr<float>(); p.rstd = rstd.data_ptr<float>();
  p.run_mean = running_mean.data_ptr<float>(); p.run_var = running_var.data_ptr<float>();
  p.nbt = reinterpret_cast<long long*>(num_batches_tracked.data_ptr<int64_t>());
  p.eps = (float)eps; p.momentum = (float)momentum;
  c10::cuda::CUDAGuard guard(z.device());
  launch_colsum(p, false, ticket, z);
}

// H [rows, >= C] bf16 = dropout(relu(gamma (Z - mean_s) rstd_s + beta)); drop_p > 0: the mask of dropout_philox at
// (drop_state, drop_layer, row, column)
void bn_fwd_apply(const at::Tensor& z, int64_t C, const std::vector<int64_t>& offs, const at::Tensor& mean, const at::Tensor& rstd,
                  const at::Tensor& gamma, const at::Tensor& beta, const at::Tensor& h, const c10::optional<at::Tensor>& drop_state,
                  double drop_p, int64_t drop_layer) {
  TORCH_CHECK(C > 0 && C % 8 == 0, "batch norm width must be a multiple of 8");
  const int rows = (int)z.size(0);
  check_rows(z, at::kFloat, rows, (int)C, "z");
  check_rows(h, at::kBFloat16, rows, (int)C, "h");
  for (const at::Tensor* t : {&mean, &rstd, &gamma, &beta}) check_f32(*t, "mean / rstd / gamma / beta");
  BnApplyParams p;
  std::memset(&p, 0, sizeof(p));
  p.g = make_segs(offs, rows);
  TORCH_CHECK(mean.numel() >= p.g.nseg * C && rstd.numel() >= p.g.nseg * C && gamma.numel() == C && beta.numel() == C);
  p.z = z.data_ptr<float>(); p.ldz = (int)z.stride(0);
  p.mean = mean.data_ptr<float>(); p.rstd = rstd.data_ptr<float>();
  p.gamma = gamma.data_ptr<float>(); p.beta = beta.data_ptr<float>();
  p.h = reinterpret_cast<__nv_bfloat16*>(h.data_ptr()); p.ldh = (int)h.stride(0);
  p.rows = rows; p.C = (int)C; p.groups = (int)((C + 31) / 32 * 4);
  TORCH_CHECK(drop_p >= 0.0 && drop_p < 1.0, "dropout rate must be in [0, 1), got ", drop_p);
  if (drop_p > 0.0) {
    TORCH_CHECK(drop_state.has_value() && drop_state->defined() && drop_state->is_cuda() &&
                drop_state->scalar_type() == at::kLong && drop_state->numel() >= 2 &&
                (reinterpret_cast<uintptr_t>(drop_state->data_ptr()) & 15) == 0, "drop_state must be a 16-byte aligned CUDA int64 [2]");
    TORCH_CHECK(drop_layer >= 0 && drop_layer < 256, "drop_layer must be in [0, 256)");
    p.drop_state = reinterpret_cast<const unsigned long long*>(drop_state->data_ptr());
    p.drop_thr = (uint32_t)std::llround(drop_p * 65536.0);
    p.drop_scale = (float)(1.0 / (1.0 - drop_p));
    p.drop_layer = (uint32_t)drop_layer;
  }
  if (rows == 0) return;
  c10::cuda::CUDAGuard guard(z.device());
  const long long n = (long long)rows * p.groups;
  bn_apply_kernel<<<(unsigned)((n + kBnThreads - 1) / kBnThreads), kBnThreads, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// Backward sums: gsum [nseg, 2, C] = per segment (sum dY, sum dY x^); dgamma += sum over segments of sum dY x^, dbeta +=
// sum over segments of sum dY
void bn_bwd_reduce(const at::Tensor& dy, const at::Tensor& z, int64_t C, const std::vector<int64_t>& offs, const at::Tensor& ticket,
                   const at::Tensor& mean, const at::Tensor& rstd, const at::Tensor& gsum, const at::Tensor& dgamma,
                   const at::Tensor& dbeta) {
  TORCH_CHECK(C > 0 && C % 8 == 0, "batch norm width must be a multiple of 8");
  const int rows = (int)z.size(0);
  check_rows(z, at::kFloat, rows, (int)C, "z");
  check_rows(dy, at::kBFloat16, rows, (int)C, "dy");
  for (const at::Tensor* t : {&mean, &rstd, &gsum, &dgamma, &dbeta}) check_f32(*t, "mean / rstd / gsum / dgamma / dbeta");
  BnSumParams p;
  std::memset(&p, 0, sizeof(p));
  p.g = make_segs(offs, rows);
  TORCH_CHECK(mean.numel() >= p.g.nseg * C && rstd.numel() >= p.g.nseg * C && gsum.numel() >= 2 * p.g.nseg * C &&
              dgamma.numel() == C && dbeta.numel() == C);
  p.z = z.data_ptr<float>(); p.ldz = (int)z.stride(0);
  p.dy = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()); p.lddy = (int)dy.stride(0);
  p.C = (int)C;
  p.mean = mean.data_ptr<float>(); p.rstd = rstd.data_ptr<float>();
  p.gsum = gsum.data_ptr<float>(); p.dgamma = dgamma.data_ptr<float>(); p.dbeta = dbeta.data_ptr<float>();
  c10::cuda::CUDAGuard guard(z.device());
  launch_colsum(p, true, ticket, z);
}

// dZ [rows, >= C] bf16 = gamma rstd_s (dY - gsum_s[0] / n_s - x^ gsum_s[1] / n_s)
void bn_bwd_apply(const at::Tensor& dy, const at::Tensor& z, int64_t C, const std::vector<int64_t>& offs, const at::Tensor& mean,
                  const at::Tensor& rstd, const at::Tensor& gamma, const at::Tensor& gsum, const at::Tensor& dz) {
  TORCH_CHECK(C > 0 && C % 8 == 0, "batch norm width must be a multiple of 8");
  const int rows = (int)z.size(0);
  check_rows(z, at::kFloat, rows, (int)C, "z");
  check_rows(dy, at::kBFloat16, rows, (int)C, "dy");
  check_rows(dz, at::kBFloat16, rows, (int)C, "dz");
  for (const at::Tensor* t : {&mean, &rstd, &gamma, &gsum}) check_f32(*t, "mean / rstd / gamma / gsum");
  BnBwdParams p;
  std::memset(&p, 0, sizeof(p));
  p.g = make_segs(offs, rows);
  TORCH_CHECK(mean.numel() >= p.g.nseg * C && rstd.numel() >= p.g.nseg * C && gsum.numel() >= 2 * p.g.nseg * C && gamma.numel() == C);
  p.z = z.data_ptr<float>(); p.ldz = (int)z.stride(0);
  p.dy = reinterpret_cast<const __nv_bfloat16*>(dy.data_ptr()); p.lddy = (int)dy.stride(0);
  p.mean = mean.data_ptr<float>(); p.rstd = rstd.data_ptr<float>(); p.gamma = gamma.data_ptr<float>(); p.gsum = gsum.data_ptr<float>();
  p.dz = reinterpret_cast<__nv_bfloat16*>(dz.data_ptr()); p.lddz = (int)dz.stride(0);
  p.rows = rows; p.C = (int)C;
  if (rows == 0) return;
  c10::cuda::CUDAGuard guard(z.device());
  const long long n = (long long)rows * (C / 8);
  bn_bwd_apply_kernel<<<(unsigned)((n + kBnThreads - 1) / kBnThreads), kBnThreads, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace glb
