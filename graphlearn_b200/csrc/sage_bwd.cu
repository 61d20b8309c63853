// Backward of the fused GraphSAGE layer on the Hopper tensor cores (warpgroup MMA, wgmma).
//
//   dW_l [n_out, K_total] += dZ_l^T . A_l          (reduction over the 10^4..10^5 destination rows of the layer)
//
// Both operands are row-major with the REDUCTION index outermost, i.e. exactly the "MN-major" (transposed) operand
// form of wgmma: a [64 rows x 64 cols] bf16 slab is one SWIZZLE_128B atom column (K = row index), so the
// tiles are staged with plain coalesced 16-byte loads + swizzled 16-byte shared stores - no transpose.
//
// Split-K over the whole chip: CTA (block, split) owns a [128 x <=128] block of dW and a contiguous range
// of rows; it accumulates in registers (fp32) over its rows and adds the partial block to the flat gradient
// buffer with vectorised red.global.add (the gradient buffer is zeroed once per step).
//
// The dZ operand is usually not read but COMPUTED on the fly (fused "backward through ReLU + mean
// aggregation"):
//     dZ_l[r, :] = relu'(H_l[r, :]) * ( dA_{l+1}[self row of r, 0:d]  +  scale * dA_{l+1}[parent of r, kp_self : kp_self + d] )
// so dZ of the big hop segments never exists in HBM for 2-layer models; the bias gradient (column sums of
// dZ) falls out of the same registers.  Deeper models can ask for dZ to be written (needed by dA = dZ.W).
// The instantiation ROUTE = true serves the other aggregations of the layer above: a per-segment self scale (gcn:
// both parts are scaled by 1 / (k + 1)) and, for max, the argmax bytes of the parent row, which pass column c of the
// neighbour part only to the child j = (r - row0) % k that held the maximum:
//     dZ_l[r, c] = relu'(H_l[r, c]) * ( sscale * self[c]  +  scale * [amax[parent][c] == j] * nbr[c] )
//
// sage_bwd_dz_kernel is the dZ-only mode of the same body (DW = false, no `a` / `dw`): the producers compute and store dZ
// to dz_out and nothing else runs (no A loads, no MMAs) - the batch-normalised layer's dY, whose dW follows from the
// normalised gradient on the dense-dZ path.
//
// warps 0..15 : producers (loads -> ReLU-grad math -> swizzled st.shared) and, as four warpgroups, the MMA issuers:
//               warpgroup g owns the [64 x 64] quadrant (rows 64 (g & 1), columns 64 (g >> 1)) of the CTA's dW block
//               and issues its MMAs of a stage once all 16 warps have filled it (3-stage mbarrier ring, operands of
//               stage st+1 already in flight in registers; a stage is released once wgmma.wait_group reports its
//               MMAs complete); the epilogue adds the register accumulators with red.global
//
// Reference semantics: plain autograd of EgoSAGEConv (graphlearn/python/nn/tf/layers/ego_sage_conv.py:71-106).
#include <torch/extension.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <cstring>
#include "host_utils.h"
#include "gmma.cuh"

namespace glb {

constexpr int kDwProdWarps = 16;
constexpr int kDwProdThreads = kDwProdWarps * 32;     // 512
constexpr int kDwThreads = kDwProdThreads;            // warp 0 doubles as the MMA issuer (17 warps would round up to 20
                                                      // in the register allocator and cap the kernel at 96 registers)
constexpr int kDwStages = 3;
constexpr int kDwRows = 64;                           // reduction rows per stage (4 MMA K-steps)
constexpr int kDwZBytes = kDwRows * 128 * 2;          // dZ slab  [64 rows x 128 cols] bf16 = 16 KB
constexpr int kDwCols = 128;                          // dW columns per CTA (the register accumulators of 4 warpgroups)
constexpr int kDwBBytes = kDwRows * kDwCols * 2;      // A slab   [64 rows x 128 cols] bf16 = 16 KB
constexpr int kDwStageBytes = kDwZBytes + kDwBBytes;
constexpr int kDwMaxSegs = 4;

struct BwdSeg {
  int row0, row1;                  // rows [row0, row1) of this layer's activation buffer
  const __nv_bfloat16* self_src;   // dA_{l+1} rows aligned with row0 (row r -> self_src + (r - row0) * ld_da), or null
  const __nv_bfloat16* nbr_src;    // dA_{l+1} rows of the parents (row r -> nbr_src + ((r - row0) / k) * ld_da + nbr_col0), or null
  int k;
  float scale;
};

struct DwParams {
  const __nv_bfloat16* dz; int ld_dz;       // dense dZ (top layer) or null -> computed from the fields below
  const __nv_bfloat16* h; int ld_h;         // activations of this layer (ReLU mask) or null (no mask)
  BwdSeg seg[kDwMaxSegs]; int nseg;
  int ld_da, nbr_col0;
  __nv_bfloat16* dz_out; int ld_dz_out;     // optional materialised dZ
  const __nv_bfloat16* a; int ld_a;         // saved [self || agg] rows, [rows, n_cols]
  float* dw; int ld_dw;                     // fp32 [n_out, n_cols], accumulated
  float* dbias;                             // optional fp32 [n_out], accumulated
  int rows, n_out, dz_cols, n_cols;
  int m_blocks, n_blocks, rows_per_split;
  uint32_t lbo, sbo, kadv;                  // MN-major descriptor fields (bytes)
  // ROUTE instantiation only (after the fields above, whose offsets stay put): per segment, the self part's scale and
  // the argmax rows of the parents (row r -> amax[seg] + ((r - row0) / k) * ld_amax, one byte per column) or null
  float self_scale[kDwMaxSegs];
  const uint8_t* amax[kDwMaxSegs]; int ld_amax;
};

__device__ __forceinline__ uint4 ldg16(const void* p) { return *reinterpret_cast<const uint4*>(p); }

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

// byte offset of the 16-byte chunk (row r in [0,64), 8-column chunk c) inside an MN-major SW128 slab whose
// 64-column groups are 8 KB apart
__device__ __forceinline__ uint32_t mn_off(int r, int c) {
  return (uint32_t)(c >> 3) * 8192u + (uint32_t)(r >> 3) * 1024u + (uint32_t)(r & 7) * 128u + (uint32_t)(((c & 7) ^ (r & 7)) << 4);
}

template <bool ROUTE, bool DW>
__device__ __forceinline__ void sage_bwd_dw_body(const DwParams& p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (gmma::smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* stages = smem;
  float* colsum = reinterpret_cast<float*>(stages + kDwStages * kDwStageBytes);   // [128]
  uint64_t* bars = reinterpret_cast<uint64_t*>(colsum + 128);
  uint64_t* bar_full = bars;                    // [kDwStages] producers -> MMA
  uint64_t* bar_empty = bars + kDwStages;       // [kDwStages] MMA -> producers

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int blk = blockIdx.x % (p.m_blocks * p.n_blocks);
  const int split = blockIdx.x / (p.m_blocks * p.n_blocks);
  const int mb = blk % p.m_blocks, nb = blk / p.m_blocks;
  const int r_begin = split * p.rows_per_split;
  const int r_end = min(p.rows, r_begin + p.rows_per_split);
  const int n_steps = (r_end - r_begin + kDwRows - 1) / kDwRows;
  const int ncols_blk = min(kDwCols, p.n_cols - nb * kDwCols);  // multiple of 16

  if (tid == 0) {
    for (int i = 0; i < kDwStages; ++i) { gmma::mbar_init(bar_full + i, kDwProdWarps); gmma::mbar_init(bar_empty + i, kDwProdWarps); }
    gmma::fence_barrier_init();
  }
  if (tid < 128) colsum[tid] = 0.f;
  __syncthreads();

  const int wg = warp >> 2, wq = warp & 3;
  const int mh = wg & 1, nh = wg >> 1;            // this warpgroup's quadrant of the [128 x 128] block
  const bool wg_active = nh * 64 < ncols_blk;     // warp-uniform: a narrow block leaves the right half idle
  float acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0.f;
  {
    // ------------------------------------------------------------------ producers
    const int pt = tid;                              // 0..511
    const int zc = pt & 15, zr = pt >> 4;            // dZ slab: 16 chunks per row, rows zr and zr + 32
    const int bc = pt & 15, br = pt >> 4;            // A slab : 16 chunks per row, rows br + 32 i
    const int zcol = mb * 128 + zc * 8;              // first dZ column of this thread's chunk
    const int bcol = nb * kDwCols + bc * 8;
    const bool zcol_ok = zcol < p.dz_cols;
    const bool bcol_ok = bcol < p.n_cols;
    const bool want_out = p.dz_out != nullptr && nb == 0;
    float cs[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) cs[i] = 0.f;
    const uint4 zero4 = make_uint4(0u, 0u, 0u, 0u);
    // register-staged operands of one 64-row stage; two sets are alive so that the loads of stage st+1 are in
    // flight while stage st is converted and stored (the kernel is bound by bytes in flight, not by math)
    // (ROUTE: am = argmax bytes of the chunk's 8 columns, j = this row's index among its parent's children; rows without
    // an argmax keep am = 0, j = 0, which passes every column)
    struct StageRegs { uint4 bv[2], hv[2], sv[2], nv[2]; float nscale[2]; uint2 am[2]; uint32_t j[2]; float sscale[2]; };
    auto issue = [&](int st, StageRegs& g) {
      const int rbase = r_begin + st * kDwRows;
      if constexpr (DW) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = rbase + br + 32 * i;
          g.bv[i] = (r < r_end && bcol_ok) ? ldg16(p.a + (size_t)r * p.ld_a + bcol) : zero4;
        }
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int r = rbase + zr + 32 * i;
        g.hv[i] = zero4; g.sv[i] = zero4; g.nv[i] = zero4; g.nscale[i] = 0.f;
        if constexpr (ROUTE) { g.am[i] = make_uint2(0u, 0u); g.j[i] = 0u; g.sscale[i] = 1.f; }
        if (r < r_end && zcol_ok) {
          if (p.dz) {
            g.sv[i] = ldg16(p.dz + (size_t)r * p.ld_dz + zcol);
          } else {
            int sg = 0;
#pragma unroll
            for (int j = 1; j < kDwMaxSegs; ++j) if (j < p.nseg && r >= p.seg[j].row0) sg = j;
            const BwdSeg& q = p.seg[sg];
            const int rl = r - q.row0;
            if (q.self_src) g.sv[i] = ldg16(q.self_src + (size_t)rl * p.ld_da + zcol);
            if (q.nbr_src) { g.nv[i] = ldg16(q.nbr_src + (size_t)(rl / q.k) * p.ld_da + p.nbr_col0 + zcol); g.nscale[i] = q.scale; }
            if constexpr (ROUTE) {
              g.sscale[i] = p.self_scale[sg];
              const uint8_t* am = p.amax[sg];
              if (am) {
                const int par = rl / q.k;
                g.am[i] = *reinterpret_cast<const uint2*>(am + (size_t)par * p.ld_amax + zcol);
                g.j[i] = (uint32_t)(rl - par * q.k);
              }
            }
            if (p.h) g.hv[i] = ldg16(p.h + (size_t)r * p.ld_h + zcol);
          }
        }
      }
    };
    auto process = [&](int st, StageRegs& g) {
      const int s = st % kDwStages;
      const int rbase = r_begin + st * kDwRows;
      // math: dZ = relu'(h) * (self + scale * nbr)
      uint4 zv[2];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        if (p.dz) { zv[i] = g.sv[i]; continue; }
        const uint32_t* ps = reinterpret_cast<const uint32_t*>(&g.sv[i]);
        const uint32_t* pn = reinterpret_cast<const uint32_t*>(&g.nv[i]);
        const uint32_t* ph = reinterpret_cast<const uint32_t*>(&g.hv[i]);
        uint32_t o[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float2 a = unpack_bf16x2(ps[j]), b = unpack_bf16x2(pn[j]);
          float gx, gy;
          if constexpr (ROUTE) {
            const uint32_t w = j < 2 ? g.am[i].x : g.am[i].y;            // bytes of columns 2 j, 2 j + 1
            const uint32_t sh = 16 * (j & 1);
            const float nx = ((w >> sh) & 0xFFu) == g.j[i] ? b.x : 0.f, ny = ((w >> (sh + 8)) & 0xFFu) == g.j[i] ? b.y : 0.f;
            gx = a.x * g.sscale[i] + nx * g.nscale[i]; gy = a.y * g.sscale[i] + ny * g.nscale[i];
          } else {
            gx = a.x + b.x * g.nscale[i]; gy = a.y + b.y * g.nscale[i];
          }
          if (p.h) {
            const float2 hh = unpack_bf16x2(ph[j]);
            if (!(hh.x > 0.f)) gx = 0.f;
            if (!(hh.y > 0.f)) gy = 0.f;
          }
          o[j] = pack_bf16x2(gx, gy);
          cs[2 * j] += gx; cs[2 * j + 1] += gy;
        }
        zv[i] = make_uint4(o[0], o[1], o[2], o[3]);
        const int r = rbase + zr + 32 * i;
        if (want_out && r < r_end && zcol < p.ld_dz_out) *reinterpret_cast<uint4*>(p.dz_out + (size_t)r * p.ld_dz_out + zcol) = zv[i];
      }
      if constexpr (!DW) return;
      gmma::mbar_wait(bar_empty + s, (uint32_t)(((st / kDwStages) & 1) ^ 1));
      uint8_t* zs = stages + (size_t)s * kDwStageBytes;
      uint8_t* bs = zs + kDwZBytes;
#pragma unroll
      for (int i = 0; i < 2; ++i) *reinterpret_cast<uint4*>(zs + mn_off(zr + 32 * i, zc)) = zv[i];
#pragma unroll
      for (int i = 0; i < 2; ++i) *reinterpret_cast<uint4*>(bs + mn_off(br + 32 * i, bc)) = g.bv[i];
      gmma::fence_proxy_async_smem();
      __syncwarp();
      if (lane == 0) gmma::mbar_arrive(bar_full + s);
      // MMA issue for this stage (the operands of the next stage are already in flight in this warp's registers)
      gmma::mbar_wait(bar_full + s, (uint32_t)((st / kDwStages) & 1));
      if (wg_active) {
        const uint32_t zb = gmma::smem_u32(zs) + (uint32_t)mh * 8192u;         // dZ columns 64 mh .. (mn_off's group stride)
        const uint32_t bb = gmma::smem_u32(bs) + (uint32_t)nh * 8192u;         // A columns 64 nh ..
        gmma::wgmma_fence();
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4)
          gmma::mma_m64n64_bf16<1, 1>(acc, gmma::make_desc_sw128_mn(zb + k4 * p.kadv, p.lbo, p.sbo),
                                       gmma::make_desc_sw128_mn(bb + k4 * p.kadv, p.lbo, p.sbo), 1u);
        gmma::wgmma_commit();
        gmma::wgmma_wait<1>();                            // the MMAs of stage st-1 have completed
      }
      if (st > 0) {
        __syncwarp();
        if (lane == 0) gmma::mbar_arrive(bar_empty + (st - 1) % kDwStages);
      }
    };
    StageRegs ra, rb;
    if (n_steps > 0) issue(0, ra);
    for (int st = 0; st < n_steps; st += 2) {
      if (st + 1 < n_steps) issue(st + 1, rb);
      process(st, ra);
      if (st + 1 < n_steps) {
        if (st + 2 < n_steps) issue(st + 2, ra);
        process(st + 1, rb);
      }
    }
    // bias gradient = column sums of the computed dZ (only the n-block-0 CTAs of an m-block contribute): the two
    // rows of a warp are folded with a shuffle, every warp parks its 128 sums in the (now idle) stage memory and
    // 128 threads add the 16 rows up - no shared-memory atomics (they were 32-way same-address conflicts)
    if constexpr (DW) {
      gmma::wgmma_wait<0>();
      gmma::fence_regs(acc);
    }
    const bool do_bias = p.dbias && !p.dz && nb == 0 && n_steps > 0;
    if (do_bias) {
#pragma unroll
      for (int i = 0; i < 8; ++i) cs[i] += __shfl_xor_sync(0xffffffffu, cs[i], 16);
      // every warpgroup's MMAs must have completed before the stage memory is reused
      __syncthreads();
      float* wsum = reinterpret_cast<float*>(stages) + warp * 128;
      if (lane < 16) {
        *reinterpret_cast<float4*>(wsum + zc * 8) = make_float4(cs[0], cs[1], cs[2], cs[3]);
        *reinterpret_cast<float4*>(wsum + zc * 8 + 4) = make_float4(cs[4], cs[5], cs[6], cs[7]);
      }
    }
  }
  __syncthreads();
  if (p.dbias && !p.dz && nb == 0 && tid < 128 && mb * 128 + tid < p.n_out && n_steps > 0) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < kDwProdWarps; ++w) v += reinterpret_cast<const float*>(stages)[w * 128 + tid];
    atomicAdd(p.dbias + mb * 128 + tid, v);
  }
  // ------------------------------------------------------------------ epilogue: registers -> red.global.add into dW
  if (DW && n_steps > 0 && wg_active) {
    const int r0 = mh * 64 + wq * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = nh * 64 + 8 * j + 2 * (lane & 3);
      if (c < ncols_blk) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = mb * 128 + r0 + 8 * h;
          if (m < p.n_out) red_add_v2(p.dw + (size_t)m * p.ld_dw + nb * kDwCols + c, acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

template <bool ROUTE>
__global__ void __launch_bounds__(kDwThreads, 1) sage_bwd_dw_kernel(const __grid_constant__ DwParams p) {
  sage_bwd_dw_body<ROUTE, true>(p);
}

template <bool ROUTE>
__global__ void __launch_bounds__(kDwThreads, 1) sage_bwd_dz_kernel(const __grid_constant__ DwParams p) {
  sage_bwd_dw_body<ROUTE, false>(p);
}

static const __nv_bfloat16* bf16_ptr(const at::Tensor& t) { return reinterpret_cast<const __nv_bfloat16*>(t.data_ptr()); }

template <bool ROUTE, bool DW>
static void launch_dw(const DwParams& p, int grid, size_t smem) {
  static bool attr_done = false;
  auto* kernel = DW ? sage_bwd_dw_kernel<ROUTE> : sage_bwd_dz_kernel<ROUTE>;
  if (!attr_done) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_done = true;
  }
  kernel<<<grid, kDwThreads, smem, at::cuda::getCurrentCUDAStream()>>>(p);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

// dW (+)= dZ^T A with dZ either dense (`dz`) or computed from (h, segments of dA_next).
//   a = dw = None: only dZ, computed from (h, segments of dA_next), is written to dz_out ([rows, >= n_out]), nothing else
//   segs: rows [row0, row1) of the layer; self_src[i] / nbr_src[i] are views into dA_next (or None)
//   seg_self_scale: [] (all 1) or the self part's scale per segment (gcn above: 1 / (k + 1))
//   amax_src: [] or per segment None / the uint8 argmax rows of the parents (max above; aligned with nbr_src[i], >= n_out
//             columns, row stride a multiple of 8): the neighbour part of column c reaches only the child that held its max
void sage_bwd_dw(const c10::optional<at::Tensor>& dz, const c10::optional<at::Tensor>& h,
                 const std::vector<int64_t>& seg_row0, const std::vector<int64_t>& seg_row1,
                 const std::vector<c10::optional<at::Tensor>>& self_src, const std::vector<c10::optional<at::Tensor>>& nbr_src,
                 const std::vector<int64_t>& seg_k, const std::vector<double>& seg_scale, int64_t nbr_col0,
                 const c10::optional<at::Tensor>& dz_out, const c10::optional<at::Tensor>& a_opt,
                 const c10::optional<at::Tensor>& dw_opt, const c10::optional<at::Tensor>& dbias, int64_t n_out,
                 const std::vector<double>& seg_self_scale, const std::vector<c10::optional<at::Tensor>>& amax_src) {
  const bool want_dw = a_opt.has_value() && a_opt->defined();
  TORCH_CHECK(want_dw == (dw_opt.has_value() && dw_opt->defined()), "sage_bwd_dw: pass both a and dw, or neither");
  DwParams p;
  std::memset(&p, 0, sizeof(p));
  bool route = false;
  p.n_out = (int)n_out;
  if (want_dw) {
    const at::Tensor& a = *a_opt;
    const at::Tensor& dw = *dw_opt;
    TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kBFloat16 && a.dim() == 2 && a.stride(1) == 1 && a.stride(0) % 8 == 0);
    TORCH_CHECK(dw.is_cuda() && dw.scalar_type() == at::kFloat && dw.dim() == 2 && dw.stride(1) == 1 && dw.size(0) >= n_out &&
                dw.size(1) == a.size(1) && dw.stride(0) % 4 == 0 && (reinterpret_cast<uintptr_t>(dw.data_ptr()) & 15) == 0,
                "dw must be fp32 [n_out, K_total], 16-byte aligned rows");
    p.rows = (int)a.size(0); p.n_cols = (int)a.size(1);
    TORCH_CHECK(p.n_cols % 16 == 0, "K_total must be a multiple of 16");
    p.a = bf16_ptr(a); p.ld_a = (int)a.stride(0);
    p.dw = dw.data_ptr<float>(); p.ld_dw = (int)dw.stride(0);
  } else {
    TORCH_CHECK(dz_out.has_value() && dz_out->defined() && !(dz.has_value() && dz->defined()) && !(dbias.has_value() && dbias->defined()),
                "sage_bwd_dw without a / dw computes the routed dZ into dz_out only (no dz, no dbias)");
    p.rows = (int)dz_out->size(0);
  }
  const at::Tensor& dev_t = want_dw ? *a_opt : *dz_out;
  TORCH_CHECK(dev_t.is_cuda());
  c10::cuda::CUDAGuard guard(dev_t.device());
  if (dbias.has_value() && dbias->defined()) {
    TORCH_CHECK(dbias->scalar_type() == at::kFloat && dbias->numel() >= n_out);
    p.dbias = dbias->data_ptr<float>();
  }
  if (dz.has_value() && dz->defined()) {
    TORCH_CHECK(dz->scalar_type() == at::kBFloat16 && dz->dim() == 2 && dz->stride(1) == 1 && dz->size(0) == p.rows &&
                dz->stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(dz->data_ptr()) & 15) == 0);
    p.dz = bf16_ptr(*dz); p.ld_dz = (int)dz->stride(0);
    p.dz_cols = (int)(dz->stride(0) >= (n_out + 7) / 8 * 8 ? (n_out + 7) / 8 * 8 : dz->size(1) / 8 * 8);
    TORCH_CHECK(p.dz_cols >= n_out || dz->size(1) % 8 == 0, "dense dZ rows must be readable in 16-byte chunks");
  } else {
    const int nseg = (int)seg_row0.size();
    TORCH_CHECK(nseg >= 1 && nseg <= kDwMaxSegs && (int)seg_row1.size() == nseg && (int)self_src.size() == nseg &&
                (int)nbr_src.size() == nseg && (int)seg_k.size() == nseg && (int)seg_scale.size() == nseg);
    p.nseg = nseg;
    p.nbr_col0 = (int)nbr_col0;
    TORCH_CHECK(n_out % 8 == 0 && nbr_col0 % 8 == 0, "hidden width must be a multiple of 8");
    p.dz_cols = (int)n_out;
    TORCH_CHECK(want_dw || seg_row1[nseg - 1] <= p.rows, "sage_bwd_dw: the segments run past dz_out's rows");
    for (int i = 0; i < nseg; ++i) {
      BwdSeg& g = p.seg[i];
      g.row0 = (int)seg_row0[i]; g.row1 = (int)seg_row1[i]; g.k = (int)std::max<int64_t>(seg_k[i], 1); g.scale = (float)seg_scale[i];
      for (int which = 0; which < 2; ++which) {
        const auto& src = which == 0 ? self_src[i] : nbr_src[i];
        if (!(src.has_value() && src->defined())) continue;
        TORCH_CHECK(src->scalar_type() == at::kBFloat16 && src->dim() == 2 && src->stride(1) == 1 && src->stride(0) % 8 == 0 &&
                    (reinterpret_cast<uintptr_t>(src->data_ptr()) & 15) == 0);
        TORCH_CHECK(p.ld_da == 0 || p.ld_da == src->stride(0), "all dA views must share the leading dimension");
        p.ld_da = (int)src->stride(0);
        if (which == 0) { TORCH_CHECK(src->size(0) >= g.row1 - g.row0); g.self_src = bf16_ptr(*src); }
        else { TORCH_CHECK(src->size(0) * g.k >= g.row1 - g.row0); g.nbr_src = bf16_ptr(*src); }
      }
    }
    TORCH_CHECK(seg_self_scale.empty() || (int)seg_self_scale.size() == nseg, "seg_self_scale: one entry per segment");
    TORCH_CHECK(amax_src.empty() || (int)amax_src.size() == nseg, "amax_src: one entry per segment");
    for (int i = 0; i < nseg; ++i) {
      p.self_scale[i] = seg_self_scale.empty() ? 1.f : (float)seg_self_scale[i];
      route = route || p.self_scale[i] != 1.f;
      if (amax_src.empty() || !(amax_src[i].has_value() && amax_src[i]->defined())) continue;
      const at::Tensor& m = *amax_src[i];
      TORCH_CHECK(m.is_cuda() && m.scalar_type() == at::kByte && m.dim() == 2 && m.stride(1) == 1 && m.size(1) >= n_out &&
                  m.stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(m.data_ptr()) & 7) == 0 &&
                  m.size(0) * p.seg[i].k >= p.seg[i].row1 - p.seg[i].row0,
                  "amax_src[i] must be 8-byte aligned uint8 [parents, >= n_out] rows with a row stride multiple of 8");
      TORCH_CHECK(p.ld_amax == 0 || p.ld_amax == m.stride(0), "all argmax views must share the row stride");
      p.ld_amax = (int)m.stride(0);
      p.amax[i] = reinterpret_cast<const uint8_t*>(m.data_ptr());
      route = true;
    }
    if (h.has_value() && h->defined()) {
      TORCH_CHECK(h->scalar_type() == at::kBFloat16 && h->dim() == 2 && h->stride(1) == 1 && h->size(0) >= p.rows &&
                  h->size(1) >= n_out && h->stride(0) % 8 == 0 && (reinterpret_cast<uintptr_t>(h->data_ptr()) & 15) == 0);
      p.h = bf16_ptr(*h); p.ld_h = (int)h->stride(0);
    }
    if (dz_out.has_value() && dz_out->defined()) {
      TORCH_CHECK(dz_out->scalar_type() == at::kBFloat16 && dz_out->dim() == 2 && dz_out->stride(1) == 1 && dz_out->size(0) >= p.rows &&
                  dz_out->stride(0) % 8 == 0 && dz_out->size(1) >= n_out);
      p.dz_out = reinterpret_cast<__nv_bfloat16*>(dz_out->data_ptr()); p.ld_dz_out = (int)dz_out->stride(0);
    }
  }
  if (p.rows == 0) return;
  p.m_blocks = (p.n_out + 127) / 128;
  p.n_blocks = want_dw ? (p.n_cols + kDwCols - 1) / kDwCols : 1;
  const int blocks = p.m_blocks * p.n_blocks;
  const int sms = sm_count();
  const int max_splits = std::max(1, sms / blocks);
  int rps = (p.rows + max_splits - 1) / max_splits;
  rps = std::max(kDwRows, (rps + kDwRows - 1) / kDwRows * kDwRows);
  p.rows_per_split = rps;
  const int splits = (p.rows + rps - 1) / rps;
  p.lbo = 8192; p.sbo = 1024; p.kadv = 2048;
  const size_t smem = 1024 + (size_t)kDwStages * kDwStageBytes + 512 + 2 * kDwStages * 8;
  if (!want_dw) {
    if (route) launch_dw<true, false>(p, blocks * splits, smem);
    else launch_dw<false, false>(p, blocks * splits, smem);
  } else if (route) {
    launch_dw<true, true>(p, blocks * splits, smem);
  } else {
    launch_dw<false, true>(p, blocks * splits, smem);
  }
}

// ------------------------------------------------------------------------------------------------
// dA = dZ . W of every layer l >= 2, straight from the layer's forward weight images (no W^T copy), on warp-level
// mma.sync m16n8k16 (bf16 in, fp32 accumulate).  The reduction runs over the R = n_imgs * N rows of the images: image i
// holds the weight rows [i N, i N + N), zero beyond n_out.  CTA (kb, y) stages the 64-column block kb of every image,
// [R rows x 64 K columns] SW128 = R * 128 bytes, and its 4 warps each multiply 16 dZ rows with it: A fragments of 4
// reduction steps in flight, the accumulators of all 64 output columns in registers.  The B fragments come from the block by
// ldmatrix.trans: each 8x8 matrix is 8 consecutive block rows at one 16-byte chunk, which the swizzle spreads over 8
// different bank groups (N is a multiple of 8, so the images' swizzle atoms line up in the concatenated block).
// grid = (B, min(ceil(rows / 64), kDaCtasPerSm * SMs / B)) x 128 threads, B = the 64-column blocks computed (all K_total / 64
// of them, or those of at most two windows [lo0, lo0 + n0) and [lo1, ...)): when there are more row blocks than that, a CTA
// keeps its W block and walks row blocks y, y + gridDim.y, ... (a wide layer's block is up to 64 KB, and re-staging it for
// every 64 rows would cost more L2 traffic than the dZ rows themselves).
constexpr int kDaThreads = 128;
constexpr int kDaMaxR = 512;
constexpr int kDaCtasPerSm = 4;

__global__ void __launch_bounds__(kDaThreads) sage_bwd_da_kernel(const __nv_bfloat16* __restrict__ dz, int ld_dz, int rows,
                                                                 const uint8_t* __restrict__ w_img, int N, int n_imgs, int nkb,
                                                                 int lo0, int n0, int lo1,
                                                                 __nv_bfloat16* __restrict__ da, int ld_da, float alpha) {
  extern __shared__ __align__(128) uint8_t sW[];
  const int kb = (int)blockIdx.x < n0 ? lo0 + (int)blockIdx.x : lo1 + ((int)blockIdx.x - n0);
  const int R = n_imgs * N;
  const uint32_t w_base = gmma::smem_u32(sW);
  // the W block arrives by cp.async, overlapped with the first dZ loads
  for (int i = 0; i < n_imgs; ++i) {
    const uint8_t* src = w_img + ((size_t)i * nkb + kb) * N * 128;
    for (int j = threadIdx.x; j < N * 8; j += kDaThreads)
      asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(w_base + (uint32_t)(i * N * 128 + j * 16)), "l"(src + j * 16));
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  bool staged = false;
  for (int rb = blockIdx.y; rb * 64 + warp * 16 < rows || !staged; rb += gridDim.y) {
    const bool live = rb * 64 + warp * 16 < rows;                // warp-uniform
    const int r0 = rb * 64 + warp * 16 + g, r1 = r0 + 8;
    const bool ok0 = live && r0 < rows, ok1 = live && r1 < rows;
    // A fragment of reduction step ks: bf16 pairs 8 ks + t (+ 4) = dZ columns 16 ks + 2 t, + 1 (+ 8); loaded 4 steps at a
    // time, the next 4 in flight while the current 4 are multiplied
    const uint32_t* z0 = reinterpret_cast<const uint32_t*>(dz + (size_t)(ok0 ? r0 : 0) * ld_dz);
    const uint32_t* z1 = reinterpret_cast<const uint32_t*>(dz + (size_t)(ok1 ? r1 : 0) * ld_dz);
    auto load = [&](int ks0, uint32_t (&a)[4][4]) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int ks = ks0 + j;
        const bool in = 16 * ks < R;
        a[j][0] = in && ok0 ? __ldg(z0 + 8 * ks + t) : 0u;
        a[j][1] = in && ok1 ? __ldg(z1 + 8 * ks + t) : 0u;
        a[j][2] = in && ok0 ? __ldg(z0 + 8 * ks + t + 4) : 0u;
        a[j][3] = in && ok1 ? __ldg(z1 + 8 * ks + t + 4) : 0u;
      }
    };
    uint32_t a[4][4], an[4][4];
    load(0, a);
    if (!staged) {
      asm volatile("cp.async.wait_all;" ::: "memory");
      __syncthreads();
      staged = true;
      if (!live) break;
    }
    float acc[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.f;
    for (int ks0 = 0; ks0 < R / 16; ks0 += 4) {
      if (ks0 + 4 < R / 16) load(ks0 + 4, an);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (16 * (ks0 + j) < R) {
#pragma unroll
          for (int c0 = 0; c0 < 4; ++c0) {
            uint32_t b[4];
            const uint32_t row = (uint32_t)(16 * (ks0 + j) + (lane & 15)), col = (uint32_t)(16 * c0 + (lane >> 4) * 8);
            asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
                         : "=r"(b[0]), "=r"(b[1]), "=r"(b[2]), "=r"(b[3]) : "r"(w_base + gmma::sw128_offset(row, col)));
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float* c = acc[2 * c0 + h];
              asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
                           "{%0, %1, %2, %3};"
                           : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                           : "r"(a[j][0]), "r"(a[j][1]), "r"(a[j][2]), "r"(a[j][3]), "r"(b[2 * h]), "r"(b[2 * h + 1]));
            }
          }
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) a[j][q] = an[j][q];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = kb * 64 + 8 * j + 2 * t;
      if (ok0) *reinterpret_cast<uint32_t*>(da + (size_t)r0 * ld_da + c) = pack_bf16x2(acc[j][0] * alpha, acc[j][1] * alpha);
      if (ok1) *reinterpret_cast<uint32_t*>(da + (size_t)r1 * ld_da + c) = pack_bf16x2(acc[j][2] * alpha, acc[j][3] * alpha);
    }
  }
}

// dA [rows, K_total] = alpha * dZ [rows, >= R] . W with W given as its n_imgs forward (K-major SW128) images of N output
// columns each ([n_imgs][K_total / 64][N][64], zero rows beyond the real outputs), R = n_imgs * N; dZ columns [n_out, R)
// must be zero or finite.  alpha scales the fp32 accumulators before the bf16 store (alpha = 1 is exact): 1 / (1 - p)
// when the layer's input was dropped out with rate p, which leaves dZ itself unscaled for the weight gradient.
// kb_ranges: empty = every 64-column block of dA; else at most two disjoint half-open ranges [lo, hi) of blocks, and only
// their columns are written (the learned input embedding's layer 1 needs the gradient of E's columns, not the features').
void sage_bwd_da(const at::Tensor& dz, const at::Tensor& w_img, int64_t N, int64_t n_imgs, const at::Tensor& da, double alpha,
                 const std::vector<std::pair<int64_t, int64_t>>& kb_ranges) {
  const int64_t R = n_imgs * N;
  TORCH_CHECK(N % 8 == 0 && N >= 8 && n_imgs >= 1 && R % 32 == 0 && R <= kDaMaxR,
              "sage_bwd_da needs n_imgs images of N output columns (N a multiple of 8), n_imgs * N a multiple of 32 in [32, ",
              kDaMaxR, "]");
  TORCH_CHECK(dz.is_cuda() && dz.scalar_type() == at::kBFloat16 && dz.dim() == 2 && dz.stride(1) == 1 && dz.size(1) >= R &&
              dz.stride(0) % 2 == 0 && (reinterpret_cast<uintptr_t>(dz.data_ptr()) & 3) == 0,
              "dz must be a 4-byte aligned bf16 [rows, >= n_imgs * N] view with an even row stride");
  const int64_t rows = dz.size(0), k_total = da.size(1);
  TORCH_CHECK(da.is_cuda() && da.scalar_type() == at::kBFloat16 && da.dim() == 2 && da.size(0) == rows && da.stride(1) == 1 &&
              da.stride(0) % 2 == 0 && (reinterpret_cast<uintptr_t>(da.data_ptr()) & 3) == 0 && k_total % 64 == 0 && k_total >= 64,
              "da must be a 4-byte aligned bf16 [rows, K_total] view, K_total a multiple of 64");
  TORCH_CHECK(w_img.is_cuda() && w_img.scalar_type() == at::kBFloat16 && w_img.is_contiguous() && w_img.numel() == k_total * R &&
              (reinterpret_cast<uintptr_t>(w_img.data_ptr()) & 15) == 0,
              "w_img must be the 16-byte aligned [n_imgs][K_total / 64][N][64] images");
  TORCH_CHECK(rows < (int64_t)INT32_MAX / 2, "too many rows");
  if (rows == 0) return;
  c10::cuda::CUDAGuard guard(dz.device());
  static bool attr_done = false;
  if (!attr_done) {
    C10_CUDA_CHECK(cudaFuncSetAttribute(sage_bwd_da_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDaMaxR * 128));
    attr_done = true;
  }
  const int64_t nkb = k_total / 64, row_blocks = (rows + 63) / 64;
  TORCH_CHECK(kb_ranges.size() <= 2, "sage_bwd_da takes at most two column-block ranges");
  for (const auto& r : kb_ranges)
    TORCH_CHECK(0 <= r.first && r.first < r.second && r.second <= nkb, "sage_bwd_da: column-block range [", r.first, ", ",
                r.second, ") is empty or outside the ", nkb, " blocks of da");
  TORCH_CHECK(kb_ranges.size() < 2 || kb_ranges[0].second <= kb_ranges[1].first || kb_ranges[1].second <= kb_ranges[0].first,
              "sage_bwd_da: the column-block ranges overlap");
  const int64_t lo0 = kb_ranges.empty() ? 0 : kb_ranges[0].first;
  const int64_t n0 = kb_ranges.empty() ? nkb : kb_ranges[0].second - lo0;
  const int64_t lo1 = kb_ranges.size() < 2 ? 0 : kb_ranges[1].first;
  const int64_t blocks = n0 + (kb_ranges.size() < 2 ? 0 : kb_ranges[1].second - lo1);
  const dim3 grid((unsigned)blocks, (unsigned)std::min<int64_t>(row_blocks, std::max<int64_t>(1, kDaCtasPerSm * sm_count() / blocks)));
  sage_bwd_da_kernel<<<grid, kDaThreads, (size_t)R * 128, at::cuda::getCurrentCUDAStream()>>>(
      bf16_ptr(dz), (int)dz.stride(0), (int)rows, reinterpret_cast<const uint8_t*>(w_img.data_ptr()), (int)N, (int)n_imgs,
      (int)nkb, (int)lo0, (int)n0, (int)lo1, reinterpret_cast<__nv_bfloat16*>(da.data_ptr()), (int)da.stride(0), (float)alpha);
  C10_CUDA_KERNEL_LAUNCH_CHECK();
}

}  // namespace glb
