// K6 (GAT flavour): fused gather + multi-head attention aggregation over a fixed fan-out neighbourhood.
//
// EgoGATConv (graphlearn/python/nn/tf/layers/ego_gat_conv.py:89-117), per head h:
//     x' = W_x x + b_x,  n'_j = W_n n_j + b_n,  e_j = LeakyReLU( a_h . [x' || n'_j] + b_a ),  coef = softmax_j(e),
//     ret_h = sum_j coef_j n'_j,      out = mean_h ret_h
// Because the attention logit is LINEAR in the raw rows, it only needs two d_in-vectors per head
//     e_j = LeakyReLU( u_x,h . x  +  u_n,h . n_j  +  c_h ),   u_x,h = W_x,h^T a_x,h,  u_n,h = W_n,h^T a_n,h,
// and because sum_j coef_j = 1 the projection commutes with the aggregation:
//     ret_h = W_n,h ( sum_j coef_j n_j ) + b_n,h .
// So the layer is: THIS kernel (rows pulled straight from the local / peer-mapped feature shards, one online-softmax
// pass, H attention-weighted sums of the RAW rows -> bf16 A [M, H * kp]) followed by ONE wgmma GEMM with the
// concatenated W_n,h (K = H * kp) on the persistent kernel of sage_fused.cu - the [M*k, H*D] projected neighbour
// tensor of the reference never exists.
//
// The backward kernel re-gathers the rows and turns dA (= dOut . W_cat / H, a GEMM) into the gradients of u_n, the
// per-row sums d(e_self) (-> u_x, c) and, for dense inputs, dX.
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cfloat>
#include <cstring>
#include "gather_common.cuh"

namespace glb {

constexpr int kGatMaxH = 4;

struct GatParams {
  TableView tself, tnbr;
  const int64_t* self_vids;      // [M] or null (identity self_base + m)
  const int64_t* nbr_vids;       // [M, k] or null (identity nbr_base + m * k + j)
  int64_t self_base, nbr_base;
  int M, k, H;
  int kp;                        // padded neighbour width (A has H * kp columns)
  const float* u_x;              // [H, d_self]
  const float* u_n;              // [H, d_nbr]
  const float* c;                // [H]
  float slope;
  __nv_bfloat16* a_out;          // [M, H * kp]   (forward)
  float* e_out;                  // [M, k, H] leaky-relu'd logits   (forward: written, backward: read)
  float* stat;                   // [M, H, 2] running max / sum of the softmax
  int wshift_self, wshift_nbr;
  const char* zero_row;
  // backward
  const __nv_bfloat16* dA;       // [M, H * kp]
  float* du_n;                   // [H, d_nbr] accumulated
  float* dsx;                    // [M, H]  d loss / d (u_x . x + c)
  float* dx_nbr;                 // optional [M * k, d_nbr] fp32 (dense inputs)
};

template <typename T> __device__ __forceinline__ T group_sum(T v, int lanes) {
  for (int o = lanes >> 1; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// one lane group (lanes_row lanes) per destination row; rpi rows per warp
template <int DT>
__global__ void __launch_bounds__(256) gat_agg_fwd_kernel(const GatParams p) {
  constexpr int VEC = Chunk<DT>::kVec;
  const int lane = threadIdx.x & 31;
  const int lanes_row = p.kp / VEC;                       // <= 32
  const int lshift = 31 - __clz(lanes_row);
  const int rpi = 32 >> lshift;
  const int sub = lane >> lshift, lig = lane & (lanes_row - 1);
  const int f0 = lig * VEC;
  const size_t coff = (size_t)lig * 16;
  const int d_self = p.tself.dim, d_nbr = p.tnbr.dim;
  const uint32_t nbr_rb = (uint32_t)p.tnbr.stride * (DT == 0 ? 4u : 2u), self_rb = (uint32_t)p.tself.stride * (DT == 0 ? 4u : 2u);
  const int H = p.H, k = p.k;
  // this lane's slices of the projection vectors
  float ux[kGatMaxH][VEC], un[kGatMaxH][VEC];
#pragma unroll
  for (int h = 0; h < kGatMaxH; ++h)
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      ux[h][i] = (h < H && f0 + i < d_self) ? __ldg(p.u_x + h * d_self + f0 + i) : 0.f;
      un[h][i] = (h < H && f0 + i < d_nbr) ? __ldg(p.u_n + h * d_nbr + f0 + i) : 0.f;
    }
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) >> lshift;
  for (int64_t m = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> lshift); m < (int64_t)((p.M + rpi - 1) / rpi) * rpi; m += groups) {
    const bool ok = m < p.M;
    (void)sub;
    // ---- self logit
    float sx[kGatMaxH];
    {
      float xv[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) xv[i] = 0.f;
      if (ok && f0 < d_self) {
        const int64_t vid = p.self_vids ? __ldg(p.self_vids + m) : p.self_base + m;
        Chunk<DT> r; r.load(vid_ptr(p.tself, vid, p.wshift_self, self_rb, p.zero_row) + coff); r.get(xv);
      }
#pragma unroll
      for (int h = 0; h < kGatMaxH; ++h) {
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < VEC; ++i) s += ux[h][i] * xv[i];
        sx[h] = group_sum(s, lanes_row) + (h < H ? __ldg(p.c + h) : 0.f);
      }
    }
    // ---- one pass over the neighbours: online softmax + weighted sums of the raw rows
    float mx[kGatMaxH], ls[kGatMaxH], acc[kGatMaxH][VEC];
#pragma unroll
    for (int h = 0; h < kGatMaxH; ++h) {
      mx[h] = -FLT_MAX; ls[h] = 0.f;
#pragma unroll
      for (int i = 0; i < VEC; ++i) acc[h][i] = 0.f;
    }
    for (int j0 = 0; j0 < k; j0 += 4) {
      Chunk<DT> raw[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int j = j0 + u < k ? j0 + u : k - 1;
        const int64_t idx = (int64_t)(ok ? m : 0) * k + j;
        const int64_t vid = ok ? (p.nbr_vids ? __ldg(p.nbr_vids + idx) : p.nbr_base + idx) : -1;
        raw[u].load((f0 < d_nbr ? vid_ptr(p.tnbr, vid, p.wshift_nbr, nbr_rb, p.zero_row) : p.zero_row) + (f0 < d_nbr ? coff : 0));
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (j0 + u >= k) continue;
        float nv[VEC];
        raw[u].get(nv);
#pragma unroll
        for (int i = 0; i < VEC; ++i) if (f0 + i >= d_nbr) nv[i] = 0.f;
#pragma unroll
        for (int h = 0; h < kGatMaxH; ++h) {
          if (h >= H) continue;
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < VEC; ++i) s += un[h][i] * nv[i];
          float e = group_sum(s, lanes_row) + sx[h];
          e = e > 0.f ? e : e * p.slope;
          if (ok && lig == 0 && p.e_out) p.e_out[((size_t)m * k + (j0 + u)) * H + h] = e;
          const float nm = fmaxf(mx[h], e);
          const float sc = __expf(mx[h] - nm), w = __expf(e - nm);
          ls[h] = ls[h] * sc + w;
#pragma unroll
          for (int i = 0; i < VEC; ++i) acc[h][i] = acc[h][i] * sc + w * nv[i];
          mx[h] = nm;
        }
      }
    }
    if (!ok) continue;
#pragma unroll
    for (int h = 0; h < kGatMaxH; ++h) {
      if (h >= H) continue;
      const float inv = ls[h] > 0.f ? 1.f / ls[h] : 0.f;
      __nv_bfloat16* dst = p.a_out + (size_t)m * H * p.kp + h * p.kp + f0;
      if constexpr (VEC == 8) {
        uint4 o;
        o.x = pack_bf16x2(acc[h][0] * inv, acc[h][1] * inv); o.y = pack_bf16x2(acc[h][2] * inv, acc[h][3] * inv);
        o.z = pack_bf16x2(acc[h][4] * inv, acc[h][5] * inv); o.w = pack_bf16x2(acc[h][6] * inv, acc[h][7] * inv);
        *reinterpret_cast<uint4*>(dst) = o;
      } else {
        uint2 o;
        o.x = pack_bf16x2(acc[h][0] * inv, acc[h][1] * inv); o.y = pack_bf16x2(acc[h][2] * inv, acc[h][3] * inv);
        *reinterpret_cast<uint2*>(dst) = o;
      }
      if (lig == 0 && p.stat) { p.stat[((size_t)m * H + h) * 2] = mx[h]; p.stat[((size_t)m * H + h) * 2 + 1] = ls[h]; }
    }
  }
}

// backward: per destination row m and head h
//   dcoef_j = <dA_h(m), n_j>,   coef_j = exp(e_j - max) / sum,   S = sum_j coef_j dcoef_j
//   de_j = coef_j (dcoef_j - S) * leaky'(e_j)
//   du_n,h += sum_j de_j n_j      dsx_h(m) = sum_j de_j      dX_nbr[m, j] = sum_h (coef_j dA_h(m) + de_j u_n,h)
template <int DT>
__global__ void __launch_bounds__(256) gat_agg_bwd_kernel(const GatParams p) {
  constexpr int VEC = Chunk<DT>::kVec;
  extern __shared__ float s_du[];                         // [H * kp] block-level partial sums of du_n
  const int lane = threadIdx.x & 31;
  const int lanes_row = p.kp / VEC;
  const int lshift = 31 - __clz(lanes_row);
  const int rpi = 32 >> lshift;
  const int lig = lane & (lanes_row - 1);
  const int f0 = lig * VEC;
  const size_t coff = (size_t)lig * 16;
  const int d_nbr = p.tnbr.dim;
  const uint32_t nbr_rb = (uint32_t)p.tnbr.stride * (DT == 0 ? 4u : 2u);
  const int H = p.H, k = p.k;
  for (int i = threadIdx.x; i < H * p.kp; i += blockDim.x) s_du[i] = 0.f;
  __syncthreads();
  float un[kGatMaxH][VEC], dun[kGatMaxH][VEC];
#pragma unroll
  for (int h = 0; h < kGatMaxH; ++h)
#pragma unroll
    for (int i = 0; i < VEC; ++i) {
      un[h][i] = (h < H && f0 + i < d_nbr) ? __ldg(p.u_n + h * d_nbr + f0 + i) : 0.f;
      dun[h][i] = 0.f;
    }
  const int64_t groups = ((int64_t)gridDim.x * blockDim.x) >> lshift;
  for (int64_t m = (((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> lshift); m < (int64_t)((p.M + rpi - 1) / rpi) * rpi; m += groups) {
    const bool ok = m < p.M;
    float da[kGatMaxH][VEC], S[kGatMaxH], dsum[kGatMaxH], mxv[kGatMaxH], inv[kGatMaxH];
#pragma unroll
    for (int h = 0; h < kGatMaxH; ++h) {
      S[h] = 0.f; dsum[h] = 0.f; mxv[h] = 0.f; inv[h] = 0.f;
#pragma unroll
      for (int i = 0; i < VEC; ++i) da[h][i] = 0.f;
      if (ok && h < H) {
        const __nv_bfloat16* src = p.dA + (size_t)m * H * p.kp + h * p.kp + f0;
        if constexpr (VEC == 8) {
          const uint4 u = *reinterpret_cast<const uint4*>(src);
          float2 x;
          x = unpack_bf16x2(u.x); da[h][0] = x.x; da[h][1] = x.y; x = unpack_bf16x2(u.y); da[h][2] = x.x; da[h][3] = x.y;
          x = unpack_bf16x2(u.z); da[h][4] = x.x; da[h][5] = x.y; x = unpack_bf16x2(u.w); da[h][6] = x.x; da[h][7] = x.y;
        } else {
          const uint2 u = *reinterpret_cast<const uint2*>(src);
          float2 x;
          x = unpack_bf16x2(u.x); da[h][0] = x.x; da[h][1] = x.y; x = unpack_bf16x2(u.y); da[h][2] = x.x; da[h][3] = x.y;
        }
        mxv[h] = p.stat[((size_t)m * H + h) * 2];
        const float l = p.stat[((size_t)m * H + h) * 2 + 1];
        inv[h] = l > 0.f ? 1.f / l : 0.f;
      }
    }
    // pass 1: S_h = sum_j coef_j <dA_h, n_j>
    for (int j = 0; j < k; ++j) {
      const int64_t idx = (int64_t)(ok ? m : 0) * k + j;
      const int64_t vid = ok ? (p.nbr_vids ? __ldg(p.nbr_vids + idx) : p.nbr_base + idx) : -1;
      Chunk<DT> r; r.load((f0 < d_nbr ? vid_ptr(p.tnbr, vid, p.wshift_nbr, nbr_rb, p.zero_row) : p.zero_row) + (f0 < d_nbr ? coff : 0));
      float nv[VEC]; r.get(nv);
#pragma unroll
      for (int i = 0; i < VEC; ++i) if (f0 + i >= d_nbr) nv[i] = 0.f;
#pragma unroll
      for (int h = 0; h < kGatMaxH; ++h) {
        if (h >= H) continue;
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < VEC; ++i) s += da[h][i] * nv[i];
        const float dcoef = group_sum(s, lanes_row);
        const float e = ok ? p.e_out[((size_t)m * k + j) * H + h] : 0.f;
        S[h] += __expf(e - mxv[h]) * inv[h] * dcoef;
      }
    }
    // pass 2: de_j, du_n, dX
    for (int j = 0; j < k; ++j) {
      const int64_t idx = (int64_t)(ok ? m : 0) * k + j;
      const int64_t vid = ok ? (p.nbr_vids ? __ldg(p.nbr_vids + idx) : p.nbr_base + idx) : -1;
      Chunk<DT> r; r.load((f0 < d_nbr ? vid_ptr(p.tnbr, vid, p.wshift_nbr, nbr_rb, p.zero_row) : p.zero_row) + (f0 < d_nbr ? coff : 0));
      float nv[VEC]; r.get(nv);
#pragma unroll
      for (int i = 0; i < VEC; ++i) if (f0 + i >= d_nbr) nv[i] = 0.f;
      float dx[VEC];
#pragma unroll
      for (int i = 0; i < VEC; ++i) dx[i] = 0.f;
#pragma unroll
      for (int h = 0; h < kGatMaxH; ++h) {
        if (h >= H) continue;
        float s = 0.f;
#pragma unroll
        for (int i = 0; i < VEC; ++i) s += da[h][i] * nv[i];
        const float dcoef = group_sum(s, lanes_row);
        const float e = ok ? p.e_out[((size_t)m * k + j) * H + h] : 0.f;
        const float coef = __expf(e - mxv[h]) * inv[h];
        const float de = ok ? coef * (dcoef - S[h]) * (e > 0.f ? 1.f : p.slope) : 0.f;
        dsum[h] += de;
#pragma unroll
        for (int i = 0; i < VEC; ++i) { dun[h][i] += de * nv[i]; dx[i] += coef * da[h][i] + de * un[h][i]; }
      }
      if (ok && p.dx_nbr && f0 < d_nbr) {
        float* o = p.dx_nbr + ((size_t)m * k + j) * d_nbr + f0;
#pragma unroll
        for (int i = 0; i < VEC; ++i) if (f0 + i < d_nbr) o[i] = dx[i];
      }
    }
    if (ok && lig == 0)
      for (int h = 0; h < H; ++h) p.dsx[(size_t)m * H + h] = dsum[h];
  }
  // block-level reduction of du_n, then one atomic per element
#pragma unroll
  for (int h = 0; h < kGatMaxH; ++h)
    if (h < H)
#pragma unroll
      for (int i = 0; i < VEC; ++i) atomicAdd(&s_du[h * p.kp + f0 + i], dun[h][i]);
  __syncthreads();
  for (int i = threadIdx.x; i < H * p.kp; i += blockDim.x) {
    const int h = i / p.kp, f = i - h * p.kp;
    if (f < d_nbr && s_du[i] != 0.f) atomicAdd(p.du_n + h * d_nbr + f, s_du[i]);
  }
}

static int log2n(int w) { int s = 0; while ((1 << s) < w) ++s; return (1 << s) == w ? s : -1; }

static void fill_common(GatParams& p, const at::Tensor& tself_desc, const c10::optional<at::Tensor>& self_vids, int64_t self_base,
                        const at::Tensor& tnbr_desc, const c10::optional<at::Tensor>& nbr_vids, int64_t nbr_base, int64_t M, int64_t k,
                        const at::Tensor& u_x, const at::Tensor& u_n, const at::Tensor& c, double slope, std::vector<at::Tensor>& keep) {
  std::memset(&p, 0, sizeof(p));
  p.tself = table_from_desc(tself_desc);
  p.tnbr = table_from_desc(tnbr_desc);
  TORCH_CHECK(p.tself.dtype == p.tnbr.dtype && (p.tnbr.dtype == 0 || p.tnbr.dtype == 1), "GAT kernel: fp32 or bf16 tables of one dtype");
  p.M = (int)M; p.k = (int)k; p.H = (int)u_n.size(0);
  TORCH_CHECK(p.H >= 1 && p.H <= kGatMaxH, "1..", kGatMaxH, " heads");
  TORCH_CHECK(u_x.is_cuda() && u_x.scalar_type() == at::kFloat && u_x.is_contiguous() && u_x.size(0) == p.H && u_x.size(1) == p.tself.dim);
  TORCH_CHECK(u_n.is_cuda() && u_n.scalar_type() == at::kFloat && u_n.is_contiguous() && u_n.size(1) == p.tnbr.dim);
  TORCH_CHECK(c.is_cuda() && c.scalar_type() == at::kFloat && c.numel() == p.H);
  const int vec = p.tnbr.dtype == 0 ? 4 : 8;
  int kp = 64;
  while (kp < std::max(p.tself.dim, p.tnbr.dim)) kp <<= 1;
  TORCH_CHECK(kp / vec <= 32, "GAT kernel: rows wider than ", 32 * vec, " elements are not supported");
  TORCH_CHECK((p.tself.stride * (p.tself.dtype == 0 ? 4 : 2)) % 16 == 0 && (p.tnbr.stride * (p.tnbr.dtype == 0 ? 4 : 2)) % 16 == 0);
  p.kp = kp;
  p.u_x = u_x.data_ptr<float>(); p.u_n = u_n.data_ptr<float>(); p.c = c.data_ptr<float>(); p.slope = (float)slope;
  p.self_base = self_base; p.nbr_base = nbr_base;
  if (self_vids.has_value() && self_vids->defined()) { auto t = self_vids->contiguous(); check_cuda_i64(t, "self_vids"); TORCH_CHECK(t.numel() == M); keep.push_back(t); p.self_vids = t.data_ptr<int64_t>(); }
  if (nbr_vids.has_value() && nbr_vids->defined()) { auto t = nbr_vids->contiguous(); check_cuda_i64(t, "nbr_vids"); TORCH_CHECK(t.numel() == M * k); keep.push_back(t); p.nbr_vids = t.data_ptr<int64_t>(); }
  p.wshift_self = log2n(p.tself.world); p.wshift_nbr = log2n(p.tnbr.world);
  static std::vector<at::Tensor> zr(64);
  const int dev = u_n.get_device();
  if (!zr[dev].defined()) zr[dev] = at::zeros({1024}, u_n.options());
  p.zero_row = reinterpret_cast<const char*>(zr[dev].data_ptr());
}

// -> (A bf16 [M, H * kp], e fp32 [M, k, H], stat fp32 [M, H, 2])
std::vector<at::Tensor> gat_agg_forward(const at::Tensor& tself_desc, const c10::optional<at::Tensor>& self_vids, int64_t self_base,
                                        const at::Tensor& tnbr_desc, const c10::optional<at::Tensor>& nbr_vids, int64_t nbr_base,
                                        int64_t M, int64_t k, const at::Tensor& u_x, const at::Tensor& u_n, const at::Tensor& c,
                                        double slope) {
  c10::cuda::CUDAGuard guard(u_n.device());
  GatParams p;
  std::vector<at::Tensor> keep;
  fill_common(p, tself_desc, self_vids, self_base, tnbr_desc, nbr_vids, nbr_base, M, k, u_x, u_n, c, slope, keep);
  auto a = at::zeros({M, (int64_t)p.H * p.kp}, u_n.options().dtype(at::kBFloat16));
  auto e = at::empty({M, k, (int64_t)p.H}, u_n.options());
  auto stat = at::empty({M, (int64_t)p.H, 2}, u_n.options());
  if (M == 0) return {a, e, stat};
  p.a_out = reinterpret_cast<__nv_bfloat16*>(a.data_ptr()); p.e_out = e.data_ptr<float>(); p.stat = stat.data_ptr<float>();
  const int vec = p.tnbr.dtype == 0 ? 4 : 8;
  const int rpi = 32 / (p.kp / vec);
  const int64_t warps = (M + rpi - 1) / rpi;
  const unsigned blocks = (unsigned)std::min<int64_t>((warps + 7) / 8, (int64_t)sm_count() * 8);
  if (p.tnbr.dtype == 0) gat_agg_fwd_kernel<0><<<blocks, 256, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  else gat_agg_fwd_kernel<1><<<blocks, 256, 0, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {a, e, stat};
}

// -> (du_n fp32 [H, d_nbr], dsx fp32 [M, H], dx_nbr fp32 [M*k, d_nbr] | undefined)
std::vector<at::Tensor> gat_agg_backward(const at::Tensor& tself_desc, const at::Tensor& tnbr_desc, const c10::optional<at::Tensor>& nbr_vids,
                                         int64_t nbr_base, int64_t M, int64_t k, const at::Tensor& u_x, const at::Tensor& u_n,
                                         const at::Tensor& c, double slope, const at::Tensor& dA, const at::Tensor& e, const at::Tensor& stat,
                                         bool want_dx) {
  c10::cuda::CUDAGuard guard(u_n.device());
  GatParams p;
  std::vector<at::Tensor> keep;
  fill_common(p, tself_desc, c10::nullopt, 0, tnbr_desc, nbr_vids, nbr_base, M, k, u_x, u_n, c, slope, keep);
  TORCH_CHECK(dA.is_cuda() && dA.scalar_type() == at::kBFloat16 && dA.is_contiguous() && dA.size(0) == M && dA.size(1) == (int64_t)p.H * p.kp);
  TORCH_CHECK(e.scalar_type() == at::kFloat && e.is_contiguous() && stat.scalar_type() == at::kFloat && stat.is_contiguous());
  auto du_n = at::zeros({(int64_t)p.H, (int64_t)p.tnbr.dim}, u_n.options());
  auto dsx = at::zeros({M, (int64_t)p.H}, u_n.options());
  at::Tensor dx;
  if (want_dx) dx = at::zeros({M * k, (int64_t)p.tnbr.dim}, u_n.options());
  if (M == 0) return {du_n, dsx, dx};
  p.dA = reinterpret_cast<const __nv_bfloat16*>(dA.data_ptr());
  p.e_out = const_cast<float*>(e.data_ptr<float>()); p.stat = const_cast<float*>(stat.data_ptr<float>());
  p.du_n = du_n.data_ptr<float>(); p.dsx = dsx.data_ptr<float>(); p.dx_nbr = want_dx ? dx.data_ptr<float>() : nullptr;
  const int vec = p.tnbr.dtype == 0 ? 4 : 8;
  const int rpi = 32 / (p.kp / vec);
  const int64_t warps = (M + rpi - 1) / rpi;
  const unsigned blocks = (unsigned)std::min<int64_t>((warps + 7) / 8, (int64_t)sm_count() * 4);
  const size_t smem = (size_t)p.H * p.kp * sizeof(float);
  if (p.tnbr.dtype == 0) gat_agg_bwd_kernel<0><<<blocks, 256, smem, at::cuda::getCurrentCUDAStream()>>>(p);
  else gat_agg_bwd_kernel<1><<<blocks, 256, smem, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
  return {du_n, dsx, dx};
}

}  // namespace glb
