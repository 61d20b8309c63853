// Peer-memory runtime + K8 (one-shot gradient all-reduce fused with cast/scale)
// + fused Adam over the flat parameter buffer.
//
// The reference moves every byte through gRPC/protobuf
// (graphlearn/src/service/dist/grpc_channel.cc:81-90) and relies on PyTorch DDP
// for the gradient all-reduce (graphlearn/examples/pytorch/gcn/train.py:192-193).
// Here every rank cudaMalloc's "symmetric" buffers, exchanges CUDA IPC handles
// once through torch.distributed and afterwards kernels simply dereference
// peer pointers over NVLink / NVSwitch.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cuda_runtime.h>
#include <cstring>
#include "host_utils.h"

namespace glb {

// ---------------------------------------------------------------------------
// symmetric heap / CUDA IPC
// ---------------------------------------------------------------------------
int64_t symm_alloc(int64_t nbytes, int64_t device) {
  c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  void* p = nullptr;
  size_t n = (size_t)((nbytes + 511) / 512 * 512);
  if (n == 0) n = 512;
  C10_CUDA_CHECK(cudaMalloc(&p, n));
  C10_CUDA_CHECK(cudaMemset(p, 0, n));
  C10_CUDA_CHECK(cudaDeviceSynchronize());
  return reinterpret_cast<int64_t>(p);
}

void symm_free(int64_t ptr, int64_t device) {
  c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  C10_CUDA_CHECK(cudaFree(reinterpret_cast<void*>(ptr)));
}

py::bytes ipc_get_handle(int64_t ptr, int64_t device) {
  c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  cudaIpcMemHandle_t h;
  C10_CUDA_CHECK(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(ptr)));
  return py::bytes(reinterpret_cast<const char*>(&h), sizeof(h));
}

int64_t ipc_open_handle(const std::string& handle, int64_t device) {
  c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  TORCH_CHECK(handle.size() == sizeof(cudaIpcMemHandle_t), "bad IPC handle size");
  cudaIpcMemHandle_t h;
  std::memcpy(&h, handle.data(), sizeof(h));
  void* p = nullptr;
  C10_CUDA_CHECK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
  return reinterpret_cast<int64_t>(p);
}

void ipc_close_handle(int64_t ptr, int64_t device) {
  c10::cuda::CUDAGuard guard((c10::DeviceIndex)device);
  C10_CUDA_CHECK(cudaIpcCloseMemHandle(reinterpret_cast<void*>(ptr)));
}

at::Tensor tensor_from_ptr(int64_t ptr, std::vector<int64_t> sizes, int64_t dtype_code, int64_t device) {
  at::ScalarType st = dtype_code == 0 ? at::kFloat : dtype_code == 1 ? at::kBFloat16
                    : dtype_code == 2 ? at::kLong : dtype_code == 3 ? at::kInt : at::kByte;
  auto opts = at::TensorOptions().dtype(st).device(at::kCUDA, (c10::DeviceIndex)device);
  return at::from_blob(reinterpret_cast<void*>(ptr), sizes, opts);
}

// ---------------------------------------------------------------------------
// K8: one-shot all-reduce over peer memory
// ---------------------------------------------------------------------------
constexpr int kArMaxBlocks = 256;

struct AllReduceParams {
  PeerTableMut stage;        // per rank: float [2][n_pad]   (double buffered staging, symmetric)
  PeerTableMut flags;        // per rank: uint32 [kArMaxBlocks][kMaxWorld]  (symmetric, zero-init)
  unsigned long long* epochs;  // local: [kArMaxBlocks]
  int* error_flag;           // local: set to 1 on barrier timeout
  float* grad;               // local flat gradient (in/out)
  int64_t n;                 // elements (multiple of 4)
  int64_t n_pad;
  float scale;
  int rank, world;
};

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__global__ void __launch_bounds__(512) allreduce_oneshot_kernel(const AllReduceParams p) {
  const int b = blockIdx.x;
  const unsigned long long e = p.epochs[b] + 1;      // this call's epoch (same on every rank)
  const int parity = (int)(e & 1);
  const int64_t per_block = ((p.n / 4 + gridDim.x - 1) / gridDim.x) * 4;
  const int64_t lo = (int64_t)b * per_block;
  const int64_t hi = min(p.n, lo + per_block);

  // phase 0: publish my slice (scaled) into my staging buffer
  float* my_stage = reinterpret_cast<float*>(p.stage.p[p.rank]) + (size_t)parity * p.n_pad;
  for (int64_t i = lo + 4 * (int64_t)threadIdx.x; i < hi; i += 4 * (int64_t)blockDim.x) {
    float4 g = *reinterpret_cast<const float4*>(p.grad + i);
    g.x *= p.scale; g.y *= p.scale; g.z *= p.scale; g.w *= p.scale;
    *reinterpret_cast<float4*>(my_stage + i) = g;
  }
  // (no per-thread system fence: the CTA barrier + the flag writers' st.release.sys order the staging stores, see adam_pack_kernel)
  __syncthreads();

  // phase 1: block-level cross-GPU barrier (block b of every rank)
  __shared__ int timed_out;
  if (threadIdx.x == 0) timed_out = 0;
  __syncthreads();
  if (threadIdx.x < p.world) {
    const int r = threadIdx.x;
    unsigned int* remote = reinterpret_cast<unsigned int*>(p.flags.p[r]) + b * kMaxWorld + p.rank;
    st_release_sys(remote, (unsigned int)e);
    const unsigned int* mine = reinterpret_cast<const unsigned int*>(p.flags.p[p.rank]) + b * kMaxWorld + r;
    long long t0 = clock64();
    while ((int)(ld_acquire_sys(mine) - (unsigned int)e) < 0) {
      if (clock64() - t0 > 20000000000LL) { *p.error_flag = 1; timed_out = 1; break; }   // ~10 s watchdog
    }
  }
  __syncthreads();
  if (timed_out) {
    // a peer died or diverged: ABORT - the local gradient stays untouched (never reduce half-written staging
    // buffers); the sticky error flag makes the fused optimiser skip its update and PeerAllReduce.check() raise
    if (threadIdx.x == 0) p.epochs[b] = e;
    return;
  }

  // phase 2: pull + reduce every rank's slice straight from peer HBM
  for (int64_t i = lo + 4 * (int64_t)threadIdx.x; i < hi; i += 4 * (int64_t)blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int r = 0; r < kMaxWorld; ++r) {
      if (r < p.world) {
        const float4* src = reinterpret_cast<const float4*>(
            reinterpret_cast<const float*>(p.stage.p[r]) + (size_t)parity * p.n_pad + i);
        float4 v = __ldcv(src);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
    }
    *reinterpret_cast<float4*>(p.grad + i) = acc;
  }
  if (threadIdx.x == 0) p.epochs[b] = e;
}

// desc (CPU int64): [rank, world, n_pad, stage_ptr[8], flags_ptr[8]]
void allreduce_oneshot(const at::Tensor& desc, const at::Tensor& grad, const at::Tensor& epochs,
                       const at::Tensor& error_flag, double scale) {
  TORCH_CHECK(desc.device().is_cpu() && desc.scalar_type() == at::kLong && desc.numel() == 3 + 2 * kMaxWorld);
  TORCH_CHECK(grad.is_cuda() && grad.scalar_type() == at::kFloat && grad.is_contiguous());
  TORCH_CHECK(epochs.is_cuda() && epochs.scalar_type() == at::kLong && epochs.numel() >= kArMaxBlocks);
  TORCH_CHECK(error_flag.is_cuda() && error_flag.scalar_type() == at::kInt);
  c10::cuda::CUDAGuard guard(grad.device());
  const int64_t* d = desc.data_ptr<int64_t>();
  AllReduceParams p;
  p.rank = (int)d[0]; p.world = (int)d[1]; p.n_pad = d[2];
  for (int r = 0; r < kMaxWorld; ++r) {
    p.stage.p[r] = reinterpret_cast<void*>(d[3 + r]);
    p.flags.p[r] = reinterpret_cast<void*>(d[3 + kMaxWorld + r]);
  }
  p.n = grad.numel();
  TORCH_CHECK(p.n % 4 == 0 && p.n <= p.n_pad, "flat grad must be padded to a multiple of 4 and fit the staging buffer");
  TORCH_CHECK((reinterpret_cast<uintptr_t>(grad.data_ptr()) & 15) == 0);
  p.grad = grad.data_ptr<float>();
  p.epochs = reinterpret_cast<unsigned long long*>(epochs.data_ptr<int64_t>());
  p.error_flag = error_flag.data_ptr<int>();
  p.scale = (float)scale;
  // grid MUST be identical on every rank (slices are matched by block index)
  int blocks = (int)std::min<int64_t>(kArMaxBlocks, std::max<int64_t>(1, p.n / (4 * 512)));
  allreduce_oneshot_kernel<<<blocks, 512, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// ---------------------------------------------------------------------------
// fused Adam over a flat buffer; step count lives on the device (graph safe)
// ---------------------------------------------------------------------------
__global__ void step_advance_kernel(uint64_t* rng_state, long long* opt_step, uint64_t rng_inc) {
  if (rng_state) rng_state[1] += rng_inc;
  if (opt_step) opt_step[0] += 1;
}

__global__ void __launch_bounds__(256)
adam_flat_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ m,
                 float* __restrict__ v, int64_t n, const long long* __restrict__ step_ptr, float lr,
                 float beta1, float beta2, float eps, float weight_decay) {
  const float step = (float)step_ptr[0];
  const float bc1 = 1.f - powf(beta1, step);
  const float bc2 = 1.f - powf(beta2, step);
  const float step_size = lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float gi = g[i];
    float wi = w[i];
    if (weight_decay != 0.f) gi += weight_decay * wi;
    float mi = beta1 * m[i] + (1.f - beta1) * gi;
    float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
    m[i] = mi; v[i] = vi;
    float denom = sqrtf(vi) * inv_sqrt_bc2 + eps;
    w[i] = wi - step_size * mi / denom;
  }
}

// ---------------------------------------------------------------------------
// Adam fused with everything the next step needs from the parameters (engine/fast_sage.py):
//   * the gradient (and the scratch accumulators behind it) is zeroed in the same pass - no memset per step
//   * every weight matrix is re-emitted as the bf16 SWIZZLE_128B K-major image the fused forward kernel feeds
//     to wgmma and dA = dZ . W reads - no pack kernels per step
//   * the loss accumulated by the fused CE epilogue is moved to `loss_out` before it is cleared
// One thread owns 8 consecutive parameters (parameter starts are 8-aligned in the flat buffer).
// ---------------------------------------------------------------------------
constexpr int kMaxPackMats = 8;
struct PackMat {
  long long off;          // first element in the flat buffer
  int n_out, k_total;     // fp32 master [n_out, k_total]
  int N;                  // rows of ONE forward image per k-block (padded n_out, or n_out / n_imgs for N-split layers);
                          // image i holds the weight rows [i * N, i * N + N)
  uint8_t* img;           // forward image: (k_total/64) k-blocks of [N x 64] bf16, SW128
};
struct AdamPackParams {
  float* w; float* g; float* m; float* v;
  long long n;                       // parameters (multiple of 8)
  const long long* step_ptr;
  float lr, beta1, beta2, eps, weight_decay;
  float* scratch; int n_scratch;     // accumulators behind the gradients (zeroed); scratch[0] = loss
  float* loss_out;
  PackMat mats[kMaxPackMats];
  int n_mats;
  // fused one-shot peer all-reduce of the gradient (world > 1): stage -> cross-GPU flag barrier -> every rank pulls
  // all peers' slices, reduces in registers and applies Adam right away (the reduced gradient is never written back)
  PeerTableMut stage;                // per rank: [2][n_pad] fp32 (or bf16 in the same bytes), double buffered
  PeerTableMut flags;                // per rank: uint32 [kArMaxBlocks][kMaxWorld]
  unsigned long long* epochs;        // local [kArMaxBlocks]
  int* error_flag;                   // sticky: a barrier timed out -> skip every later update
  long long n_pad;
  float ar_scale;
  int rank, world, stage_bf16;
  long long* drop_ctr;               // or null: the dropout step counter of the fused trainer, advanced once per step
};

__global__ void __launch_bounds__(128) adam_pack_kernel(const __grid_constant__ AdamPackParams p) {
  const float step = (float)p.step_ptr[0];
  const float bc1 = 1.f - powf(p.beta1, step);
  const float bc2 = 1.f - powf(p.beta2, step);
  const float step_size = p.lr / bc1;
  const float inv_sqrt_bc2 = rsqrtf(bc2);
  // the step's forward launches, the only readers of the counter, precede this kernel on the stream
  if (p.drop_ctr != nullptr && blockIdx.x == 0 && threadIdx.x == 0) ++*p.drop_ctr;
  if (p.error_flag != nullptr && *p.error_flag != 0) return;          // a previous collective failed: freeze the model
  // contiguous slice of 8-element chunks per block (identical on every rank: slices are matched by block index)
  const long long chunks = p.n >> 3;
  const long long per_block = (chunks + gridDim.x - 1) / gridDim.x;
  const long long c_lo = (long long)blockIdx.x * per_block, c_hi = min(chunks, c_lo + per_block);
  unsigned long long e = 0;
  int parity = 0;
  if (p.world > 1) {
    const int b = blockIdx.x;
    e = p.epochs[b] + 1;
    parity = (int)(e & 1);
    // phase 0: publish my (scaled) slice
    if (p.stage_bf16) {
      uint4* st = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.stage.p[p.rank]) + (size_t)parity * p.n_pad);
      for (long long c = c_lo + threadIdx.x; c < c_hi; c += blockDim.x) {
        const float4 a = *reinterpret_cast<const float4*>(p.g + (c << 3)), b4 = *reinterpret_cast<const float4*>(p.g + (c << 3) + 4);
        uint4 o;
        o.x = pack_bf16x2(a.x * p.ar_scale, a.y * p.ar_scale); o.y = pack_bf16x2(a.z * p.ar_scale, a.w * p.ar_scale);
        o.z = pack_bf16x2(b4.x * p.ar_scale, b4.y * p.ar_scale); o.w = pack_bf16x2(b4.z * p.ar_scale, b4.w * p.ar_scale);
        st[c] = o;
      }
    } else {
      float4* st = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.stage.p[p.rank]) + (size_t)parity * p.n_pad);
      for (long long c = c_lo + threadIdx.x; c < c_hi; c += blockDim.x) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float4 a = *reinterpret_cast<const float4*>(p.g + (c << 3) + 4 * h);
          a.x *= p.ar_scale; a.y *= p.ar_scale; a.z *= p.ar_scale; a.w *= p.ar_scale;
          st[2 * c + h] = a;
        }
      }
    }
    // No per-thread system fence here: 128 x blocks fence.sc.sys per step cost tens of microseconds on an NVSwitch box.
    // The CTA barrier orders every thread's staging stores before the flag writers, and their st.release.sys is
    // cumulative over everything that happens-before it (PTX memory model: causality order through bar.sync).
    __shared__ int timed_out;
    if (threadIdx.x == 0) timed_out = 0;
    __syncthreads();
    // phase 1: cross-GPU barrier of block b
    if (threadIdx.x < p.world) {
      const int r = threadIdx.x;
      st_release_sys(reinterpret_cast<unsigned int*>(p.flags.p[r]) + b * kMaxWorld + p.rank, (unsigned int)e);
      const unsigned int* mine = reinterpret_cast<const unsigned int*>(p.flags.p[p.rank]) + b * kMaxWorld + r;
      const long long t0 = clock64();
      while ((int)(ld_acquire_sys(mine) - (unsigned int)e) < 0) {
        if (clock64() - t0 > 20000000000LL) { *p.error_flag = 1; timed_out = 1; break; }   // ~10 s watchdog
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) p.epochs[b] = e;
    if (timed_out) return;                                             // abort: parameters stay untouched
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    if (p.loss_out) p.loss_out[0] = p.scratch[0];
    for (int i = 0; i < p.n_scratch; ++i) p.scratch[i] = 0.f;
  }
  for (long long c = c_lo + threadIdx.x; c < c_hi; c += blockDim.x) {
    const long long i0 = c << 3;
    float w[8], g[8], m[8], v[8];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 a = *reinterpret_cast<const float4*>(p.w + i0 + 4 * h);
      const float4 cm = *reinterpret_cast<const float4*>(p.m + i0 + 4 * h), cv = *reinterpret_cast<const float4*>(p.v + i0 + 4 * h);
      w[4 * h] = a.x; w[4 * h + 1] = a.y; w[4 * h + 2] = a.z; w[4 * h + 3] = a.w;
      m[4 * h] = cm.x; m[4 * h + 1] = cm.y; m[4 * h + 2] = cm.z; m[4 * h + 3] = cm.w;
      v[4 * h] = cv.x; v[4 * h + 1] = cv.y; v[4 * h + 2] = cv.z; v[4 * h + 3] = cv.w;
    }
    if (p.world > 1) {
      // phase 2: pull + reduce this chunk straight from every peer's staging buffer
#pragma unroll
      for (int i = 0; i < 8; ++i) g[i] = 0.f;
#pragma unroll
      for (int r = 0; r < kMaxWorld; ++r) {
        if (r < p.world) {
          if (p.stage_bf16) {
            const uint4 u = __ldcv(reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p.stage.p[r]) + (size_t)parity * p.n_pad) + c);
            float2 x;
            x = unpack_bf16x2(u.x); g[0] += x.x; g[1] += x.y;
            x = unpack_bf16x2(u.y); g[2] += x.x; g[3] += x.y;
            x = unpack_bf16x2(u.z); g[4] += x.x; g[5] += x.y;
            x = unpack_bf16x2(u.w); g[6] += x.x; g[7] += x.y;
          } else {
            const float4* src = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.stage.p[r]) + (size_t)parity * p.n_pad) + 2 * c;
            const float4 a = __ldcv(src), b4 = __ldcv(src + 1);
            g[0] += a.x; g[1] += a.y; g[2] += a.z; g[3] += a.w; g[4] += b4.x; g[5] += b4.y; g[6] += b4.z; g[7] += b4.w;
          }
        }
      }
    } else {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float4 b4 = *reinterpret_cast<const float4*>(p.g + i0 + 4 * h);
        g[4 * h] = b4.x; g[4 * h + 1] = b4.y; g[4 * h + 2] = b4.z; g[4 * h + 3] = b4.w;
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      float gi = g[i];
      if (p.weight_decay != 0.f) gi += p.weight_decay * w[i];
      m[i] = p.beta1 * m[i] + (1.f - p.beta1) * gi;
      v[i] = p.beta2 * v[i] + (1.f - p.beta2) * gi * gi;
      w[i] -= step_size * m[i] / (sqrtf(v[i]) * inv_sqrt_bc2 + p.eps);
    }
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      *reinterpret_cast<float4*>(p.w + i0 + 4 * h) = make_float4(w[4 * h], w[4 * h + 1], w[4 * h + 2], w[4 * h + 3]);
      *reinterpret_cast<float4*>(p.m + i0 + 4 * h) = make_float4(m[4 * h], m[4 * h + 1], m[4 * h + 2], m[4 * h + 3]);
      *reinterpret_cast<float4*>(p.v + i0 + 4 * h) = make_float4(v[4 * h], v[4 * h + 1], v[4 * h + 2], v[4 * h + 3]);
      *reinterpret_cast<float4*>(p.g + i0 + 4 * h) = z;
    }
    // ---- weight images
    int mi = -1;
#pragma unroll
    for (int j = 0; j < kMaxPackMats; ++j)
      if (j < p.n_mats && i0 >= p.mats[j].off && i0 < p.mats[j].off + (long long)p.mats[j].n_out * p.mats[j].k_total) mi = j;
    if (mi >= 0) {
      const PackMat& pm = p.mats[mi];
      const int rel = (int)(i0 - pm.off);
      const int n = rel / pm.k_total, kcol = rel - n * pm.k_total;      // kcol is a multiple of 8: one 16-byte chunk
      uint4 val;
      val.x = pack_bf16x2(w[0], w[1]); val.y = pack_bf16x2(w[2], w[3]); val.z = pack_bf16x2(w[4], w[5]); val.w = pack_bf16x2(w[6], w[7]);
      const int kb = kcol >> 6, ch = (kcol & 63) >> 3;
      const int fi = n / pm.N, nl = n - fi * pm.N;                       // forward image index, row inside it
      const size_t off = ((size_t)fi * (pm.k_total >> 6) + kb) * pm.N * 128 + (size_t)(nl >> 3) * 1024 + (size_t)(nl & 7) * 128 +
                         (size_t)((ch ^ (nl & 7)) * 16);
      *reinterpret_cast<uint4*>(pm.img + off) = val;
    }
  }
}

// mats: CPU int64 [n_mats, 5] = (off, n_out, k_total, N, img_ptr)
// drop_ctr: optional CUDA int64 scalar incremented by one thread (the dropout step counter of the training step)
void adam_pack(const at::Tensor& w, const at::Tensor& g_store, const at::Tensor& m, const at::Tensor& v, const at::Tensor& step,
               double lr, double beta1, double beta2, double eps, double weight_decay, const c10::optional<at::Tensor>& loss_out,
               const at::Tensor& mats, const c10::optional<at::Tensor>& ar_desc, const c10::optional<at::Tensor>& ar_epochs,
               const c10::optional<at::Tensor>& ar_error, double ar_scale, bool stage_bf16,
               const c10::optional<at::Tensor>& drop_ctr) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && w.is_contiguous() && w.numel() % 8 == 0, "flat params must be padded to 8");
  TORCH_CHECK(g_store.is_cuda() && g_store.scalar_type() == at::kFloat && g_store.numel() >= w.numel() && m.numel() == w.numel() && v.numel() == w.numel());
  TORCH_CHECK(mats.device().is_cpu() && mats.scalar_type() == at::kLong && mats.dim() == 2 && mats.size(1) == 5 && mats.size(0) <= kMaxPackMats);
  c10::cuda::CUDAGuard guard(w.device());
  AdamPackParams p;
  std::memset(&p, 0, sizeof(p));
  p.w = w.data_ptr<float>(); p.g = g_store.data_ptr<float>(); p.m = m.data_ptr<float>(); p.v = v.data_ptr<float>();
  p.n = w.numel();
  p.step_ptr = reinterpret_cast<const long long*>(step.data_ptr<int64_t>());
  p.lr = (float)lr; p.beta1 = (float)beta1; p.beta2 = (float)beta2; p.eps = (float)eps; p.weight_decay = (float)weight_decay;
  p.scratch = p.g + p.n; p.n_scratch = (int)(g_store.numel() - w.numel());
  if (loss_out.has_value() && loss_out->defined()) { TORCH_CHECK(loss_out->is_cuda() && loss_out->scalar_type() == at::kFloat); p.loss_out = loss_out->data_ptr<float>(); }
  p.n_mats = (int)mats.size(0);
  const int64_t* d = mats.data_ptr<int64_t>();
  for (int i = 0; i < p.n_mats; ++i) {
    PackMat& pm = p.mats[i];
    pm.off = d[5 * i]; pm.n_out = (int)d[5 * i + 1]; pm.k_total = (int)d[5 * i + 2]; pm.N = (int)d[5 * i + 3];
    pm.img = reinterpret_cast<uint8_t*>(d[5 * i + 4]);
    TORCH_CHECK(pm.off % 8 == 0 && pm.k_total % 64 == 0, "weight matrices must start 8-aligned with K padded to 64");
  }
  p.world = 1;
  if (ar_desc.has_value() && ar_desc->defined()) {
    // desc (CPU int64): [rank, world, n_pad, stage_ptr[8], flags_ptr[8]]  (PeerAllReduce.desc)
    TORCH_CHECK(ar_desc->device().is_cpu() && ar_desc->scalar_type() == at::kLong && ar_desc->numel() == 3 + 2 * kMaxWorld);
    const int64_t* a = ar_desc->data_ptr<int64_t>();
    p.rank = (int)a[0]; p.world = (int)a[1]; p.n_pad = a[2];
    for (int r = 0; r < kMaxWorld; ++r) {
      p.stage.p[r] = reinterpret_cast<void*>(a[3 + r]);
      p.flags.p[r] = reinterpret_cast<void*>(a[3 + kMaxWorld + r]);
    }
    TORCH_CHECK(p.n <= p.n_pad && ar_epochs.has_value() && ar_epochs->numel() >= kArMaxBlocks && ar_error.has_value());
    p.epochs = reinterpret_cast<unsigned long long*>(ar_epochs->data_ptr<int64_t>());
    p.error_flag = ar_error->data_ptr<int>();
    p.ar_scale = (float)ar_scale;
    p.stage_bf16 = stage_bf16 ? 1 : 0;
  }
  if (drop_ctr.has_value() && drop_ctr->defined()) {
    TORCH_CHECK(drop_ctr->is_cuda() && drop_ctr->scalar_type() == at::kLong && drop_ctr->numel() == 1, "drop_ctr must be a CUDA int64 scalar");
    p.drop_ctr = reinterpret_cast<long long*>(drop_ctr->data_ptr<int64_t>());
  }
  if (p.n == 0) return;
  // small blocks: one 8-element chunk per thread per pass, spread over every SM; the grid depends only on n, so it
  // is identical on every rank (the fused all-reduce matches slices by block index)
  const int blocks = (int)std::min<int64_t>(kArMaxBlocks, ((p.n >> 3) + 127) / 128);
  adam_pack_kernel<<<std::max(blocks, 1), 128, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// dst[i] = src[i] (int64); src may alias pinned host memory (UVA): the engine's seed staging copy
__global__ void copy_i64_kernel(int64_t* __restrict__ dst, const int64_t* __restrict__ src, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[i];
}

void copy_i64(const at::Tensor& dst, const at::Tensor& src) {
  TORCH_CHECK(dst.is_cuda() && dst.scalar_type() == at::kLong && src.scalar_type() == at::kLong && dst.numel() == src.numel() &&
              dst.is_contiguous() && src.is_contiguous());
  c10::cuda::CUDAGuard guard(dst.device());
  const int64_t n = dst.numel();
  if (n == 0) return;
  copy_i64_kernel<<<(unsigned)((n + 255) / 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(dst.data_ptr<int64_t>(), src.data_ptr<int64_t>(), n);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void step_advance(const c10::optional<at::Tensor>& rng_state, const c10::optional<at::Tensor>& opt_step,
                  int64_t rng_inc) {
  uint64_t* rp = nullptr; long long* sp = nullptr;
  c10::Device dev(at::kCUDA, 0);
  if (rng_state.has_value()) { rp = reinterpret_cast<uint64_t*>(rng_state->data_ptr<int64_t>()); dev = rng_state->device(); }
  if (opt_step.has_value()) { sp = reinterpret_cast<long long*>(opt_step->data_ptr<int64_t>()); dev = opt_step->device(); }
  c10::cuda::CUDAGuard guard(dev);
  step_advance_kernel<<<1, 1, 0, at::cuda::getCurrentCUDAStream()>>>(rp, sp, (uint64_t)rng_inc);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

void adam_flat(const at::Tensor& w, const at::Tensor& g, const at::Tensor& m, const at::Tensor& v,
               const at::Tensor& step, double lr, double beta1, double beta2, double eps,
               double weight_decay) {
  TORCH_CHECK(w.is_cuda() && w.scalar_type() == at::kFloat && w.is_contiguous());
  TORCH_CHECK(g.numel() == w.numel() && m.numel() == w.numel() && v.numel() == w.numel());
  TORCH_CHECK(step.is_cuda() && step.scalar_type() == at::kLong);
  c10::cuda::CUDAGuard guard(w.device());
  int64_t n = w.numel();
  if (n == 0) return;
  int blocks = (int)std::min<int64_t>((int64_t)sm_count() * 4, (n + 255) / 256);
  adam_flat_kernel<<<blocks, 256, 0, at::cuda::getCurrentCUDAStream()>>>(
      w.data_ptr<float>(), g.data_ptr<float>(), m.data_ptr<float>(), v.data_ptr<float>(), n,
      reinterpret_cast<const long long*>(step.data_ptr<int64_t>()), (float)lr, (float)beta1, (float)beta2,
      (float)eps, (float)weight_decay);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace glb
