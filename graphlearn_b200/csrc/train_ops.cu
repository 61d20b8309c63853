// Fused training-step helpers for the hand-scheduled EgoGraphSAGE engine
// (engine/fast_sage.py): everything between the tensor-core GEMMs that the
// autograd path runs as ~40 tiny elementwise / reduce kernels.
//
//  * softmax_ce_kernel     logits -> mean cross-entropy loss, dlogits (bf16,
//                          already scaled by 1/B) and the bias gradient
//                          (column sums) in ONE single-CTA kernel.
// Loss parity: graphlearn/python/nn/tf/loss.py (softmax cross entropy).
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
