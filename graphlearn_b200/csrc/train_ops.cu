// Fused training-step helpers for the hand-scheduled EgoGraphSAGE engine
// (engine/fast_sage.py): everything between the tensor-core GEMMs that the
// autograd path runs as ~40 tiny elementwise / reduce kernels.
//
//  * softmax_ce_kernel     logits -> mean cross-entropy loss, dlogits (bf16,
//                          already scaled by 1/B) and the bias gradient
//                          (column sums) in ONE single-CTA kernel.
//  * link_loss_kernel      src / dst / negative embeddings -> dot-product link loss (sigmoid or sampled
//                          softmax), the gradient of every row (bf16) and the bias gradient in ONE kernel.
//  * link_roots_kernel     staged edge batch -> (src, dst) roots of a link-prediction step.
// Loss parity: graphlearn/python/nn/tf/loss.py (softmax cross entropy, sigmoid / unsupervised softmax CE).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cfloat>
#include "host_utils.h"

namespace glb {

// warp per row; 8 rows per CTA.  `labels_table[seeds[r] / world]` is the label when `seeds` is given
// (seed nodes are owned by this rank), else labels_table[r].  loss_accum / dbias must be zeroed by
// the caller (they live in the flat gradient storage that is memset once per step).
__global__ void __launch_bounds__(256)
softmax_ce_kernel(const float* __restrict__ logits, int ld_logits, const int64_t* __restrict__ labels_table,
                  const int64_t* __restrict__ seeds, int world, int B, int C, float* __restrict__ loss_accum,
                  __nv_bfloat16* __restrict__ dlogits, int ld_dl, float* __restrict__ dbias /* [C], accumulated */) {
  extern __shared__ float colsum[];      // [C]
  for (int c = threadIdx.x; c < C; c += blockDim.x) colsum[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const float invB = 1.f / (float)B;
  if (r < B) {
    const float* row = logits + (size_t)r * ld_logits;
    float mx = -FLT_MAX;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float se = 0.f;
    for (int c = lane; c < C; c += 32) se += __expf(row[c] - mx);
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const int64_t y = seeds ? labels_table[seeds[r] / world] : labels_table[r];
    const bool valid = y >= 0 && y < C;
    const float inv = 1.f / se;
    for (int c = lane; c < C; c += 32) {
      float g = valid ? (__expf(row[c] - mx) * inv - (c == y ? 1.f : 0.f)) * invB : 0.f;
      dlogits[(size_t)r * ld_dl + c] = __float2bfloat16(g);
      if (dbias) atomicAdd(&colsum[c], g);
    }
    if (lane == 0 && valid) atomicAdd(loss_accum, (mx + __logf(se) - row[y]) * invB);
  }
  __syncthreads();
  if (dbias)
    for (int c = threadIdx.x; c < C; c += blockDim.x) atomicAdd(dbias + c, colsum[c]);
}

// ---------------------------------------------------------------------------
// Link prediction (unsupervised EgoGraphSAGE, engine/fast_link_sage.py).  Rows of `emb` in root order: [0, B) src,
// [B, 2B) dst, 2B + b*n + j the j-th negative of src b.  One warp per positive edge b holds z_src (d <= 256: 8
// floats per lane), computes the n + 1 scores by shuffle reductions and writes the gradient of every row of its
// edge - each row of `demb` has exactly one writer, so no atomics except the loss and the bias column sums.
//   sigmoid: mean_b softplus(-s_b) + mean_{b,j} softplus(s_bj)       g_b = -sigma(-s_b)/B,  g_bj = sigma(s_bj)/(B n)
//   softmax: mean_b CE([s_b, s_b1..s_bn] / T, class 0)               g = (p - onehot_0) / (B T)
// Loss parity: nn/loss.py sigmoid_cross_entropy_loss / unsupervised_softmax_cross_entropy_loss.
constexpr int kLinkMaxDim = 256;

__device__ __forceinline__ void load_row8(const float* __restrict__ row, int d, int lane, float (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    v[i] = c < d ? row[c] : 0.f;
  }
}

__device__ __forceinline__ float warp_dot8(const float (&a)[8], const float (&b)[8]) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) s = fmaf(a[i], b[i], s);
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  return s;
}

__device__ __forceinline__ void store_row8(__nv_bfloat16* __restrict__ row, int d, int lane, float g, const float (&v)[8]) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int c = lane + 32 * i;
    if (c < d) row[c] = __float2bfloat16(g * v[i]);
  }
}

__device__ __forceinline__ float softplus(float x) { return fmaxf(x, 0.f) + log1pf(expf(-fabsf(x))); }

__global__ void __launch_bounds__(256)
link_loss_kernel(const float* __restrict__ emb, int ld, int B, int n, int d, int softmax, float inv_t,
                 float* __restrict__ loss_accum, __nv_bfloat16* __restrict__ demb, int ld_dz,
                 float* __restrict__ dbias /* [d], accumulated */) {
  extern __shared__ float colsum[];      // [d]
  for (int c = threadIdx.x; c < d; c += blockDim.x) colsum[c] = 0.f;
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (b < B) {
    float zs[8], zo[8], acc[8];
    load_row8(emb + (size_t)b * ld, d, lane, zs);
    load_row8(emb + (size_t)(B + b) * ld, d, lane, zo);
    const float s_pos = warp_dot8(zs, zo);
    const size_t neg0 = 2 * (size_t)B + (size_t)b * n;
    // softmax: running max / sum of exp over the n + 1 scaled scores (first pass over the negatives)
    float mx = s_pos * inv_t, se = 1.f;
    if (softmax) {
      for (int j = 0; j < n; ++j) {
        float zn[8];
        load_row8(emb + (neg0 + j) * ld, d, lane, zn);
        const float s = warp_dot8(zs, zn) * inv_t;
        if (s > mx) { se = se * expf(mx - s) + 1.f; mx = s; } else { se += expf(s - mx); }
      }
    }
    const float invB = 1.f / (float)B, invBn = invB / (float)n;
    float loss, g;
    if (softmax) {
      loss = (mx + logf(se) - s_pos * inv_t) * invB;
      g = (expf(s_pos * inv_t - mx) / se - 1.f) * inv_t * invB;
    } else {
      loss = softplus(-s_pos) * invB;
      g = -invB / (1.f + expf(s_pos));
    }
    float gsum = g;
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = g * zo[i];
    store_row8(demb + (size_t)(B + b) * ld_dz, d, lane, g, zs);
    for (int j = 0; j < n; ++j) {
      load_row8(emb + (neg0 + j) * ld, d, lane, zo);
      const float s = warp_dot8(zs, zo);
      if (softmax) {
        g = expf(s * inv_t - mx) / se * inv_t * invB;
      } else {
        loss += softplus(s) * invBn;
        g = invBn / (1.f + expf(-s));
      }
      gsum += g;
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(g, zo[i], acc[i]);
      store_row8(demb + (neg0 + j) * ld_dz, d, lane, g, zs);
    }
    store_row8(demb + (size_t)b * ld_dz, d, lane, 1.f, acc);
    if (dbias) {
      // column sum of the edge's rows: dz_src + (g_b + sum_j g_bj) z_src
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int c = lane + 32 * i;
        if (c < d) atomicAdd(&colsum[c], fmaf(gsum, zs[i], acc[i]));
      }
    }
    if (lane == 0) atomicAdd(loss_accum, loss);
  }
  __syncthreads();
  if (dbias)
    for (int c = threadIdx.x; c < d; c += blockDim.x) atomicAdd(dbias + c, colsum[c]);
}

// Roots [0, 2B) of a link-prediction step from a staged edge batch `staged` [2B + 1] (pinned host memory read
// zero-copy through its UVA address, or device memory).  The last word says what the batch holds:
//   0  staged[0, 2B) are the (src, dst) vids themselves
//   1  staged[0, B) are positions in this rank's CSR: src = row_of_edge[pos] * world + rank, dst = indices[pos]
__global__ void link_roots_kernel(int64_t* __restrict__ roots, const int64_t* __restrict__ staged, int64_t B,
                                  const int64_t* __restrict__ row_of_edge, const int64_t* __restrict__ indices,
                                  int world, int rank) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B) return;
  if (staged[2 * B] != 0) {
    const int64_t pos = staged[i];
    roots[i] = row_of_edge[pos] * world + rank;
    roots[B + i] = indices[pos];
  } else {
    roots[i] = staged[i];
    roots[B + i] = staged[B + i];
  }
}

// ---------------------------------------------------------------------------
void link_loss(const at::Tensor& emb, int64_t B, int64_t n_neg, int64_t kind, double temperature,
               const at::Tensor& loss_accum, const at::Tensor& demb, const c10::optional<at::Tensor>& dbias) {
  TORCH_CHECK(emb.is_cuda() && emb.scalar_type() == at::kFloat && emb.dim() == 2 && emb.stride(1) == 1,
              "emb must be fp32 [B * (2 + n), d] (rows may be padded)");
  TORCH_CHECK(B > 0 && n_neg > 0 && emb.size(0) == B * (2 + n_neg), "emb must have B * (2 + n_neg) rows");
  const int64_t d = emb.size(1);
  TORCH_CHECK(d > 0 && d <= kLinkMaxDim, "link_loss supports embedding widths up to ", kLinkMaxDim);
  TORCH_CHECK(kind == 0 || kind == 1, "kind must be 0 (sigmoid) or 1 (softmax)");
  TORCH_CHECK(temperature > 0, "temperature must be positive");
  TORCH_CHECK(demb.is_cuda() && demb.scalar_type() == at::kBFloat16 && demb.dim() == 2 && demb.stride(1) == 1 &&
              demb.size(0) == emb.size(0) && demb.size(1) == d, "demb must be bf16 with the shape of emb (rows may be padded)");
  TORCH_CHECK(loss_accum.is_cuda() && loss_accum.scalar_type() == at::kFloat && loss_accum.numel() >= 1);
  float* db = nullptr;
  if (dbias.has_value()) {
    TORCH_CHECK(dbias->is_cuda() && dbias->scalar_type() == at::kFloat && dbias->is_contiguous() && dbias->numel() >= d);
    db = dbias->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(emb.device());
  const int blocks = (int)((B * 32 + 255) / 256);
  link_loss_kernel<<<blocks, 256, (size_t)d * sizeof(float), at::cuda::getCurrentCUDAStream()>>>(
      emb.data_ptr<float>(), (int)emb.stride(0), (int)B, (int)n_neg, (int)d, (int)kind, (float)(1.0 / temperature),
      loss_accum.data_ptr<float>(), reinterpret_cast<__nv_bfloat16*>(demb.data_ptr()), (int)demb.stride(0), db);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void link_roots(const at::Tensor& roots, const at::Tensor& staged, const at::Tensor& row_of_edge, const at::Tensor& indices,
                int64_t world, int64_t rank) {
  check_cuda_i64(roots, "roots");
  check_cuda_i64(row_of_edge, "row_of_edge");
  check_cuda_i64(indices, "indices");
  TORCH_CHECK(staged.scalar_type() == at::kLong && staged.is_contiguous() && roots.is_contiguous());
  const int64_t B = (staged.numel() - 1) / 2;
  TORCH_CHECK(B > 0 && staged.numel() == 2 * B + 1 && roots.numel() >= 2 * B, "staged must be [2B + 1], roots at least [2B]");
  c10::cuda::CUDAGuard guard(roots.device());
  link_roots_kernel<<<(unsigned)((B + 255) / 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      roots.data_ptr<int64_t>(), staged.data_ptr<int64_t>(), B, row_of_edge.data_ptr<int64_t>(), indices.data_ptr<int64_t>(),
      (int)world, (int)rank);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void softmax_ce(const at::Tensor& logits, const at::Tensor& labels_table, const c10::optional<at::Tensor>& seeds,
                int64_t world, const at::Tensor& loss_accum, const at::Tensor& dlogits,
                const c10::optional<at::Tensor>& dbias) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.dim() == 2 && logits.stride(1) == 1);
  TORCH_CHECK(labels_table.is_cuda() && labels_table.scalar_type() == at::kLong);
  TORCH_CHECK(dlogits.scalar_type() == at::kBFloat16 && dlogits.dim() == 2 && dlogits.stride(1) == 1 && dlogits.size(0) == logits.size(0) &&
              dlogits.size(1) == logits.size(1), "dlogits must be bf16 [B, C] (rows may be padded)");
  TORCH_CHECK(loss_accum.scalar_type() == at::kFloat && loss_accum.numel() >= 1);
  c10::cuda::CUDAGuard guard(logits.device());
  int B = (int)logits.size(0), C = (int)logits.size(1);
  const int64_t* sp = nullptr;
  if (seeds.has_value()) { TORCH_CHECK(seeds->scalar_type() == at::kLong && seeds->numel() == B); sp = seeds->data_ptr<int64_t>(); }
  else TORCH_CHECK(labels_table.numel() == B);
  float* db = nullptr;
  if (dbias.has_value()) { TORCH_CHECK(dbias->scalar_type() == at::kFloat && dbias->numel() >= C); db = dbias->data_ptr<float>(); }
  int blocks = (B * 32 + 255) / 256;
  softmax_ce_kernel<<<blocks, 256, (size_t)C * sizeof(float), at::cuda::getCurrentCUDAStream()>>>(
      logits.data_ptr<float>(), (int)logits.stride(0), labels_table.data_ptr<int64_t>(), sp, (int)world, B, C, loss_accum.data_ptr<float>(),
      reinterpret_cast<__nv_bfloat16*>(dlogits.data_ptr()), (int)dlogits.stride(0), db);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace glb
