// K2: negative sampling kernels.
//
// One thread per output slot (b, j): draw a candidate destination vid - uniformly over the whole
// destination node type, or ~ weight through an inverse-CDF binary search on a global prefix-sum
// array (in-degree / node-weight distributions; replaces the reference's per-type alias tables,
// graphlearn/src/core/operator/sampler/alias_method.cc:57-123) - and reject it while it is a true
// neighbour of the source (scan of the source's adjacency row, local or peer HBM) or equal to the
// source, up to `retry` times; after that strictness is dropped like the reference
// (in_degree_negative_sampler.cc:61-98, random_negative_sampler.cc:46-58).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include "csr_view.cuh"
#include "host_utils.h"

namespace glb {

CsrView csr_from_desc(const at::Tensor& desc);   // sampling.cu

struct NegParams {
  const int64_t* src;        // [B] source vids (rows of `g`)
  int64_t* out;              // [B, k]
  const double* cum;         // [n_total] inclusive prefix sums over the concatenated shards, or null (uniform)
  const int64_t* shard_off;  // [world + 1] offsets of every rank's shard inside `cum` / the uniform range
  const uint64_t* rng;
  int64_t B;
  int64_t n_total;
  int k, retry, strict, world;
  int scan_cap;
  uint32_t salt;
};

__device__ __forceinline__ int64_t pos_to_vid(const NegParams& p, int64_t pos) {
  int owner = 0;
  while (owner + 1 < p.world && pos >= p.shard_off[owner + 1]) ++owner;
  return (pos - p.shard_off[owner]) * p.world + owner;
}

__global__ void __launch_bounds__(256) negative_sample_kernel(const CsrView g, const NegParams p) {
  int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= p.B * p.k) return;
  const int64_t b = t / p.k;
  const int64_t s = __ldg(p.src + b);
  RowRef r = csr_row(g, s);
  const int64_t scan = r.deg < p.scan_cap ? r.deg : p.scan_cap;
  int64_t cand = -1;
  for (int attempt = 0; attempt <= p.retry; ++attempt) {
    uint4 rnd = rng4(p.rng, p.salt + (uint32_t)attempt * 0x9E3779B9u, (uint64_t)t);
    int64_t pos;
    if (p.cum) {
      const double total = p.cum[p.n_total - 1];
      const double u = ((double)(((uint64_t)rnd.x << 21) ^ rnd.y) + 0.5) * (1.0 / 9007199254740992.0) * total;
      int64_t lo = 0, hi = p.n_total - 1;
      while (lo < hi) { int64_t mid = (lo + hi) >> 1; if (p.cum[mid] > u) hi = mid; else lo = mid + 1; }
      pos = lo;
    } else {
      pos = (int64_t)bounded64(rnd.x, rnd.y, (uint64_t)p.n_total);
    }
    cand = pos_to_vid(p, pos);
    if (!p.strict) break;
    bool bad = false;
    for (int64_t i = 0; i < scan; ++i)
      if (__ldg(r.indices + r.beg + i) == cand) { bad = true; break; }
    if (!bad) break;
  }
  p.out[t] = cand;
}

// `out`: optional preallocated int64 [B * k] (contiguous) the draws are written to, so that the launch allocates
// nothing and can be captured into a CUDA graph; without it a fresh [B, k] tensor is returned.
at::Tensor negative_sample(const at::Tensor& csr_desc, const at::Tensor& src, int64_t k,
                           const c10::optional<at::Tensor>& cum, const at::Tensor& shard_off, int64_t n_total,
                           bool strict,
                           int64_t retry, int64_t scan_cap, const at::Tensor& rng_state, int64_t salt,
                           const c10::optional<at::Tensor>& out_buf) {
  check_cuda_i64(src, "src");
  check_cuda_i64(shard_off, "shard_off");
  c10::cuda::CUDAGuard guard(src.device());
  CsrView g = csr_from_desc(csr_desc);
  auto s = src.contiguous();
  int64_t B = s.numel();
  at::Tensor out;
  if (out_buf.has_value()) {
    out = *out_buf;
    check_cuda_i64(out, "out");
    TORCH_CHECK(out.is_contiguous() && out.numel() == B * k, "out must be a contiguous int64 tensor of B * k elements");
  } else {
    out = at::empty({B, k}, s.options());
  }
  if (B * k == 0) return out;
  NegParams p;
  p.src = s.data_ptr<int64_t>(); p.out = out.data_ptr<int64_t>();
  at::Tensor c;
  p.cum = nullptr;
  auto so = shard_off.contiguous();
  p.world = (int)so.numel() - 1;
  TORCH_CHECK(p.world == g.world, "shard offsets must have world + 1 entries");
  p.shard_off = so.data_ptr<int64_t>();
  if (cum.has_value()) {
    c = cum->contiguous();
    TORCH_CHECK(c.is_cuda() && c.scalar_type() == at::kDouble, "cum must be a CUDA float64 tensor");
    p.cum = c.data_ptr<double>();
  }
  p.n_total = n_total;
  TORCH_CHECK(n_total > 0 && (!cum.has_value() || c.numel() == n_total), "bad candidate universe size");
  p.rng = reinterpret_cast<const uint64_t*>(rng_state.data_ptr<int64_t>());
  p.B = B; p.k = (int)k; p.retry = (int)retry; p.strict = strict ? 1 : 0; p.scan_cap = (int)scan_cap;
  p.salt = (uint32_t)salt;
  negative_sample_kernel<<<(unsigned)((B * k + 255) / 256), 256, 0, at::cuda::getCurrentCUDAStream()>>>(g, p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return out;
}

}  // namespace glb
