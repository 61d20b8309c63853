// Learned layer-1 input embedding of the fused GraphSAGE trainer (engine/fast_sage.py, learn_input_embedding=True).
//
// Layer 1 reads a trainable table E [n_rows, d] through its bf16 image, exactly as it reads a feature table.  Two kernels
// train it:
//   embed_grad_scatter_kernel : dA_1 = dZ_1 . W_1 holds, per layer-1 row m of segment i (hop pair i, i + 1), the gradient of
//                               the row's [self || aggregate] input.  The self half goes to the gradient row of hops[i][m],
//                               the neighbour half, scaled by the aggregator, to the rows of hops[i + 1][m k .. m k + k)
//                               (vector fp32 reductions); every row read by the forward gets its bit in the touched-row
//                               bitmap, ids outside the table (read as zero rows) get nothing
//   embed_lazy_adam_kernel    : one pass over the bitmap; each touched row gets torch.optim.SparseAdam's update of its
//                               moments and master row, its bf16 image row is rewritten, its gradient row zeroed and its
//                               bit cleared.  Untouched rows are never read or written.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cstring>
#include "host_utils.h"

namespace glb {

constexpr int kEmbMaxSegs = 4;
constexpr int kEmbThreads = 256;

struct EmbSeg {
  const int64_t* self_ids;       // [M] ids of hop i
  const int64_t* nbr_ids;        // [M k] ids of hop i + 1
  const __nv_bfloat16* da;       // dA_1 row m of the segment at da + m * ld_da
  const uint8_t* amax;           // max: argmax byte of each neighbour-half column (row m at amax + m * ld_amax), else null
  long long item0;               // first warp item (= layer-1 row) of the segment
  int M, k;
  float sscale, nscale;          // scale of the self half / of the neighbour half
};

struct EmbScatterParams {
  EmbSeg seg[kEmbMaxSegs];
  int nseg;
  int ld_da, nbr_col0, ld_amax;
  int chunks;                    // 4-column chunks of a gradient row
  float* grad; int ld_g;         // fp32 [n_rows, ld_g]
  uint32_t* bits;                // one bit per row
  long long n_rows, items;
};

__device__ __forceinline__ void red_add_v4(float* addr, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// one warp per layer-1 row m (item): its lanes walk the (1 + k) destination rows x `chunks` 4-column chunks
__global__ void __launch_bounds__(kEmbThreads) embed_grad_scatter_kernel(const __grid_constant__ EmbScatterParams p) {
  const int lane = threadIdx.x & 31;
  const long long nwarps = (long long)gridDim.x * (kEmbThreads / 32);
  for (long long item = ((long long)blockIdx.x * kEmbThreads + threadIdx.x) >> 5; item < p.items; item += nwarps) {
    int s = 0;
#pragma unroll
    for (int j = 1; j < kEmbMaxSegs; ++j) if (j < p.nseg && item >= p.seg[j].item0) s = j;
    const EmbSeg& g = p.seg[s];
    const int m = (int)(item - g.item0);
    const int k = g.k;
    const __nv_bfloat16* da = g.da + (size_t)m * p.ld_da;
    for (int t = lane; t < (k + 1) * p.chunks; t += 32) {
      const int r = t / p.chunks, c = t - r * p.chunks;
      const int64_t vid = r == 0 ? __ldg(g.self_ids + m) : __ldg(g.nbr_ids + (size_t)m * k + (r - 1));
      if (vid < 0 || vid >= p.n_rows) continue;                  // read as a zero row: no gradient, no bit
      const uint2 u = *reinterpret_cast<const uint2*>(da + (r == 0 ? 0 : p.nbr_col0) + 4 * c);
      const float2 a = unpack_bf16x2(u.x), b = unpack_bf16x2(u.y);
      const float sc = r == 0 ? g.sscale : g.nscale;
      float4 v = make_float4(a.x * sc, a.y * sc, b.x * sc, b.y * sc);
      if (r > 0 && g.amax != nullptr) {                          // max: only the columns whose maximum this neighbour held
        const uint32_t w = *reinterpret_cast<const uint32_t*>(g.amax + (size_t)m * p.ld_amax + 4 * c);
        const uint32_t j = (uint32_t)(r - 1);
        if ((w & 0xFFu) != j) v.x = 0.f;
        if (((w >> 8) & 0xFFu) != j) v.y = 0.f;
        if (((w >> 16) & 0xFFu) != j) v.z = 0.f;
        if ((w >> 24) != j) v.w = 0.f;
      }
      if (v.x != 0.f || v.y != 0.f || v.z != 0.f || v.w != 0.f) red_add_v4(p.grad + (size_t)vid * p.ld_g + 4 * c, v);
      if (c == 0) {
        uint32_t* word = p.bits + (vid >> 5);
        const uint32_t bit = 1u << (vid & 31);
        if ((*word & bit) == 0u) atomicOr(word, bit);
      }
    }
  }
}

struct EmbAdamParams {
  float* w; float* m; float* v; float* g; int ld;         // fp32 [n_rows, ld]
  __nv_bfloat16* img; int ld_img;                          // bf16 image [n_rows, >= 4 chunks]
  uint32_t* bits; long long n_words;
  int chunks;
  const long long* step_ptr;                               // Adam step of the dense parameters (already advanced)
  double lr, beta1, beta2;
  float eps;
};

// one warp per 32-row bitmap word: its lanes walk (set bit, chunk) pairs.  torch.optim.SparseAdam's arithmetic, op for op
// (round-to-nearest intrinsics, so that no multiply-add is contracted; the scalars are formed in double and rounded once,
// as torch rounds its Python scalars - in fp32, 1 - 0.999f alone is off by 1.3e-5):
//   dm = (g - m)(1 - b1), m += dm;  dv = (g g - v)(1 - b2), v += dv;  w += -(lr sqrt(bc2) / bc1) ((dm + m_old) / (sqrt(dv + v_old) + eps))
__global__ void __launch_bounds__(kEmbThreads) embed_lazy_adam_kernel(const __grid_constant__ EmbAdamParams p) {
  const int lane = threadIdx.x & 31;
  const double step = (double)*p.step_ptr;
  const double bc1 = 1.0 - pow(p.beta1, step), bc2 = 1.0 - pow(p.beta2, step);
  const float step_size = (float)(p.lr * sqrt(bc2) / bc1);
  const float omb1 = (float)(1.0 - p.beta1), omb2 = (float)(1.0 - p.beta2);
  const long long nwarps = (long long)gridDim.x * (kEmbThreads / 32);
  for (long long wi = ((long long)blockIdx.x * kEmbThreads + threadIdx.x) >> 5; wi < p.n_words; wi += nwarps) {
    const uint32_t word = p.bits[wi];
    if (word == 0u) continue;                                 // warp-uniform
    const int n = __popc(word);
    for (int t = lane; t < n * p.chunks; t += 32) {
      const int i = t / p.chunks, c = t - i * p.chunks;
      uint32_t rest = word;
      for (int q = 0; q < i; ++q) rest &= rest - 1u;             // drop the i lowest set bits
      const long long row = wi * 32 + (long long)(__ffs(rest) - 1);
      const size_t o = (size_t)row * p.ld + 4 * c;
      const float4 g = *reinterpret_cast<const float4*>(p.g + o);
      float4 w = *reinterpret_cast<const float4*>(p.w + o);
      float4 m = *reinterpret_cast<const float4*>(p.m + o);
      float4 v = *reinterpret_cast<const float4*>(p.v + o);
      auto upd = [&](float gi, float& wi_, float& mi, float& vi) {
        const float dm = __fmul_rn(__fsub_rn(gi, mi), omb1);
        const float dv = __fmul_rn(__fsub_rn(__fmul_rn(gi, gi), vi), omb2);
        const float numer = __fadd_rn(dm, mi), denom = __fadd_rn(__fsqrt_rn(__fadd_rn(dv, vi)), p.eps);
        mi = __fadd_rn(mi, dm);
        vi = __fadd_rn(vi, dv);
        wi_ = __fadd_rn(wi_, __fmul_rn(-step_size, __fdiv_rn(numer, denom)));
      };
      upd(g.x, w.x, m.x, v.x); upd(g.y, w.y, m.y, v.y); upd(g.z, w.z, m.z, v.z); upd(g.w, w.w, m.w, v.w);
      *reinterpret_cast<float4*>(p.w + o) = w;
      *reinterpret_cast<float4*>(p.m + o) = m;
      *reinterpret_cast<float4*>(p.v + o) = v;
      *reinterpret_cast<float4*>(p.g + o) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<uint2*>(p.img + (size_t)row * p.ld_img + 4 * c) = make_uint2(pack_bf16x2(w.x, w.y), pack_bf16x2(w.z, w.w));
    }
    __syncwarp();
    if (lane == 0) p.bits[wi] = 0u;
  }
}

static int emb_grid(long long warps) {
  const long long blocks = (warps * 32 + kEmbThreads - 1) / kEmbThreads;
  return (int)std::max<long long>(1, std::min<long long>(blocks, (long long)sm_count() * 16));
}

static void check_rows(const at::Tensor& t, const char* name, at::ScalarType dt, int64_t n_rows, int64_t width, int align) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == dt && t.dim() == 2 && t.stride(1) == 1 && t.size(0) == n_rows &&
                  t.size(1) >= width && (t.stride(0) * t.element_size()) % align == 0 &&
                  (reinterpret_cast<uintptr_t>(t.data_ptr()) & (align - 1)) == 0,
              name, ": expected a ", align, "-byte aligned [", n_rows, ", >= ", width, "] row-major view");
}

// grad (fp32 [n_rows, dp], dp a multiple of 4, 16-byte rows) += the layer-1 input gradient carried by da (dA_1, bf16
// [rows, K_total]); bits (int32 [ceil(n_rows / 32)]) |= the rows the forward read.  Per segment i: dA_1 rows
// [seg_row0[i], seg_row0[i] + M_i) belong to self_ids[i] ([M_i]) and nbr_ids[i] ([M_i k_i]); the self half starts at column
// 0 and is scaled by self_scale[i], the neighbour half at nbr_col0 and is scaled by nbr_scale[i]; amax[i] (max
// aggregation) are the forward's argmax bytes of the segment, or None.
void embed_grad_scatter(const at::Tensor& da, const std::vector<int64_t>& seg_row0, const std::vector<at::Tensor>& self_ids,
                        const std::vector<at::Tensor>& nbr_ids, const std::vector<int64_t>& seg_k,
                        const std::vector<double>& self_scale, const std::vector<double>& nbr_scale, int64_t nbr_col0,
                        const std::vector<c10::optional<at::Tensor>>& amax, const at::Tensor& grad, const at::Tensor& bits) {
  const int nseg = (int)seg_row0.size();
  TORCH_CHECK(nseg >= 1 && nseg <= kEmbMaxSegs && (int)self_ids.size() == nseg && (int)nbr_ids.size() == nseg &&
                  (int)seg_k.size() == nseg && (int)self_scale.size() == nseg && (int)nbr_scale.size() == nseg &&
                  (amax.empty() || (int)amax.size() == nseg),
              "embed_grad_scatter: one entry per segment (1..", kEmbMaxSegs, ")");
  const int64_t n_rows = grad.size(0), dp = grad.size(1);
  TORCH_CHECK(dp % 4 == 0 && dp > 0, "embed_grad_scatter: gradient rows must hold a multiple of 4 columns");
  check_rows(grad, "grad", at::kFloat, n_rows, dp, 16);
  TORCH_CHECK(grad.stride(0) == dp, "grad must be contiguous");
  TORCH_CHECK(bits.is_cuda() && bits.scalar_type() == at::kInt && bits.is_contiguous() && bits.numel() * 32 >= n_rows);
  TORCH_CHECK(da.is_cuda() && da.scalar_type() == at::kBFloat16 && da.dim() == 2 && da.stride(1) == 1 && da.stride(0) % 4 == 0 &&
                  (reinterpret_cast<uintptr_t>(da.data_ptr()) & 7) == 0 && nbr_col0 % 4 == 0 && nbr_col0 + dp <= da.size(1),
              "da must be an 8-byte aligned bf16 [rows, >= nbr_col0 + dp] view");
  c10::cuda::CUDAGuard guard(da.device());
  EmbScatterParams p;
  std::memset(&p, 0, sizeof(p));
  p.nseg = nseg; p.ld_da = (int)da.stride(0); p.nbr_col0 = (int)nbr_col0; p.chunks = (int)(dp / 4);
  p.grad = grad.data_ptr<float>(); p.ld_g = (int)dp;
  p.bits = reinterpret_cast<uint32_t*>(bits.data_ptr<int32_t>()); p.n_rows = n_rows;
  long long items = 0;
  for (int i = 0; i < nseg; ++i) {
    EmbSeg& g = p.seg[i];
    const at::Tensor& s = self_ids[i];
    const at::Tensor& nb = nbr_ids[i];
    check_cuda_i64(s, "self_ids"); check_cuda_i64(nb, "nbr_ids");
    TORCH_CHECK(s.is_contiguous() && nb.is_contiguous() && seg_k[i] >= 1 && nb.numel() == s.numel() * seg_k[i] &&
                    seg_row0[i] >= 0 && seg_row0[i] + s.numel() <= da.size(0),
                "segment ", i, ": ids must be contiguous [M] / [M k] and its rows must lie inside da");
    g.self_ids = s.data_ptr<int64_t>(); g.nbr_ids = nb.data_ptr<int64_t>();
    g.da = reinterpret_cast<const __nv_bfloat16*>(da.data_ptr()) + seg_row0[i] * da.stride(0);
    g.M = (int)s.numel(); g.k = (int)seg_k[i]; g.item0 = items;
    g.sscale = (float)self_scale[i]; g.nscale = (float)nbr_scale[i];
    items += g.M;
    if (!amax.empty() && amax[i].has_value() && amax[i]->defined()) {
      const at::Tensor& a = *amax[i];
      TORCH_CHECK(seg_k[i] <= 256, "argmax bytes hold neighbour indices below 256");
      check_rows(a, "amax", at::kByte, s.numel(), dp, 4);
      TORCH_CHECK(p.ld_amax == 0 || p.ld_amax == a.stride(0), "all amax views must share the row stride");
      p.ld_amax = (int)a.stride(0);
      g.amax = reinterpret_cast<const uint8_t*>(a.data_ptr());
    }
  }
  p.items = items;
  if (items == 0) return;
  embed_grad_scatter_kernel<<<emb_grid(items), kEmbThreads, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// Lazy Adam over the rows whose bit is set (see embed_lazy_adam_kernel): w / m / v / grad fp32 [n_rows, dp] contiguous,
// img bf16 [n_rows, >= dp] (the table layer 1 reads), bits int32 [ceil(n_rows / 32)], step the device Adam step count.
void embed_lazy_adam(const at::Tensor& w, const at::Tensor& m, const at::Tensor& v, const at::Tensor& grad, const at::Tensor& img,
                     const at::Tensor& bits, const at::Tensor& step, double lr, double beta1, double beta2, double eps) {
  const int64_t n_rows = w.size(0), dp = w.size(1);
  TORCH_CHECK(dp % 4 == 0 && dp > 0, "embed_lazy_adam: rows must hold a multiple of 4 columns");
  for (const at::Tensor* t : {&w, &m, &v, &grad}) {
    check_rows(*t, "embed_lazy_adam fp32 table", at::kFloat, n_rows, dp, 16);
    TORCH_CHECK(t->size(1) == dp && t->stride(0) == dp, "embed_lazy_adam: w, m, v and grad must be contiguous [n_rows, dp]");
  }
  check_rows(img, "img", at::kBFloat16, n_rows, dp, 8);
  TORCH_CHECK(bits.is_cuda() && bits.scalar_type() == at::kInt && bits.is_contiguous() && bits.numel() * 32 >= n_rows);
  TORCH_CHECK(step.is_cuda() && step.scalar_type() == at::kLong && step.numel() == 1, "step must be a CUDA int64 scalar");
  c10::cuda::CUDAGuard guard(w.device());
  EmbAdamParams p;
  std::memset(&p, 0, sizeof(p));
  p.w = w.data_ptr<float>(); p.m = m.data_ptr<float>(); p.v = v.data_ptr<float>(); p.g = grad.data_ptr<float>(); p.ld = (int)dp;
  p.img = reinterpret_cast<__nv_bfloat16*>(img.data_ptr()); p.ld_img = (int)img.stride(0);
  p.bits = reinterpret_cast<uint32_t*>(bits.data_ptr<int32_t>()); p.n_words = (n_rows + 31) / 32;
  p.chunks = (int)(dp / 4);
  p.step_ptr = reinterpret_cast<const long long*>(step.data_ptr<int64_t>());
  p.lr = lr; p.beta1 = beta1; p.beta2 = beta2; p.eps = (float)eps;
  if (p.n_words == 0) return;
  embed_lazy_adam_kernel<<<emb_grid(p.n_words), kEmbThreads, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace glb
