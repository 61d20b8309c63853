"""Fused GraphSAGE layer op (K6+K7): gather -> aggregate -> wgmma GEMM -> bias/ReLU.

Weights are kept in the kernel's padded K layout ``[n_out, kp_self + kp_nbr]``
(each half padded to 64/128/256/512 columns; pad columns stay zero because
their gradient is exactly zero), so one tiny kernel per step turns the fp32
master weight into the bf16 SWIZZLE_128B image the TMA engine streams into
shared memory.  CUDA path = ``csrc/sage_fused.cu`` behind an autograd Function;
the backward uses the bf16 A tile saved by the forward kernel (dW = dY^T A,
dA = dY W) - plain library GEMMs.  The portable path composes the same math
from torch ops in fp32 and doubles as the numerics oracle.

Math: EgoSAGEConv, graphlearn/python/nn/tf/layers/ego_sage_conv.py:71-106.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .. import config as _config
from ..parallel.runtime import local_table_desc, native

# "max": column-wise max over the k neighbour rows (the fused trainer and the CSR mode; `sage_layer`'s autograd op
# treats the aggregate as a sum, so it never receives "max")
MODE = {"mean": 0, "sum": 1, "gcn": 2, "max": 3}
_SMEM_LIMIT = 232448


def pad_k(d: int) -> int:
    if d <= 0:
        return 0
    for p in (64, 128, 256, 512):
        if d <= p:
            return p
    raise ValueError("fused SAGE layer supports feature dims up to 512")


def pad_n(n_out: int) -> int:
    return max(64, (n_out + 63) // 64 * 64)


def padded_dims(d_self: int, d_nbr: int, mode: str):
    kp_self = 0 if mode == "gcn" else pad_k(d_self)
    return kp_self, pad_k(d_nbr)


def fused_supported(d_self: int, d_nbr: int, n_out: int, mode: str, k: int = 0, dtype=torch.bfloat16) -> bool:
    """Whether the persistent kernel runs this layer shape: any of the four aggregators (gcn also loads the self row,
    counted in the k + 1 row pointers of an item)."""
    if mode not in MODE or max(d_self, d_nbr) > 512 or n_out > 256:
        return False
    kp_self, kp_nbr = padded_dims(d_self, d_nbr, mode)
    if k > max_fanout(max(kp_self, kp_nbr), dtype):
        return False
    return smem_fits(kp_self + kp_nbr, pad_n(n_out))


def max_fanout(kp: int, dtype=torch.bfloat16) -> int:
    """Largest fan-out the gather warps take for a half row padded to `kp`: a warp keeps the row pointers of one work
    item (1-4 destination rows, k + 1 pointers each) in a 64-entry scratch."""
    lanes_row = kp // (4 if dtype == torch.float32 else 8)
    rows_per_item = 32 // lanes_row if lanes_row < 32 else 1
    return 64 // rows_per_item - 1


def fused_layer_plan(d_self: int, d_nbr: int, out_dim: int, mode: str, k: int = 0, dtype=torch.bfloat16,
                     last: bool = False):
    """How the fused trainers run a layer's forward: ``(halves, ns, N)``.  halves = 1 is one launch over the whole padded
    K (``fused_supported``); halves = 2 is split-K, two launches of kp = K / 2 each (the self half, then the neighbour
    half, which adds the self half's fp32 partial), for a mean, sum or max layer whose K = 2 kp does not fit one CTA's
    shared memory.  ns images of N output columns each hold W (N-split); a hidden layer's ns * N must equal out_dim.
    Raises ``ValueError`` naming the limit when neither fits."""
    if mode not in MODE:
        raise ValueError("unknown aggregation %r" % (mode,))
    if max(d_self, d_nbr) > 512:
        raise ValueError("the fused GraphSAGE layer takes inputs up to 512 wide (got %d and %d)" % (d_self, d_nbr))
    kp_self, kp_nbr = padded_dims(d_self, d_nbr, mode)

    def fits(kt):
        ns, N = split_images(kt, out_dim)
        return ns, N, smem_fits(kt, N) and (ns == 1 or last or ns * N == out_dim)

    kt = kp_self + kp_nbr
    ns, N, ok = fits(kt)
    if ok and fused_supported(d_self, d_nbr, min(out_dim, N), mode, k, dtype):
        return 1, ns, N
    halves = 1
    if not smem_fits(kt, N) and mode != "gcn" and kp_self == kp_nbr:
        halves, kt = 2, kp_nbr
        ns, N, ok = fits(kt)
    what = "the fused GraphSAGE layer (%s, inputs %d + %d wide, %d outputs)" % (mode, d_self, d_nbr, out_dim)
    if not smem_fits(kt, N):
        raise ValueError("%s does not fit: a %d-column slice of W at K = %d exceeds the shared memory" % (what, N, kt))
    if not ok:
        raise ValueError("%s does not fit: hidden width %d does not split evenly over %d weight images of %d columns"
                         % (what, out_dim, ns, N))
    if k > max_fanout(max(kp_self, kp_nbr), dtype):
        raise ValueError("%s: fan-out %d exceeds the limit of %d for inputs padded to %d columns"
                         % (what, k, max_fanout(max(kp_self, kp_nbr), dtype), max(kp_self, kp_nbr)))
    if halves == 1 or N > 256:
        raise ValueError("%s does not fit: an image of %d output columns exceeds the kernel's 256" % (what, N))
    return halves, ns, N


def smem_bytes(k_total: int, n_pad: int) -> int:
    """Dynamic shared memory of the persistent kernel, term for term as csrc/sage_fused.cu sage_smem_bytes:
    alignment slack + two A tiles + W image + 19 gather warps x 64 row pointers + bias + control block."""
    nkb = k_total // 64
    return 1024 + 2 * nkb * (64 * 128) + nkb * n_pad * 128 + 19 * 64 * 8 + 256 * 4 + (5 + 2) * 8


def smem_fits(k_total: int, n_pad: int) -> bool:
    return smem_bytes(k_total, n_pad) <= _SMEM_LIMIT


def image_width(n_out: int, ns: int) -> int:
    """Padded output columns N of one forward weight image when the n_out rows of W are N-split over `ns` images."""
    return pad_n(n_out) if ns == 1 else (-(-n_out // ns) + 31) // 32 * 32


def split_images(k_total: int, n_out: int):
    """(ns, N): the fewest images (at most 8) whose W slice fits in shared memory next to the A tiles.  The caller
    checks ``smem_fits(k_total, N)``: 8 images may still be too few."""
    ns = 1
    while not smem_fits(k_total, image_width(n_out, ns)) and ns < 8:
        ns += 1
    return ns, image_width(n_out, ns)


def pack_images(weight_p: torch.Tensor, N: int, ns: int) -> torch.Tensor:
    """The `ns` bf16 SWIZZLE_128B images of a padded fp32 weight ``[n_out, k_total]``, concatenated: image i holds the
    rows [i N, i N + N) of W, zero rows beyond n_out."""
    wpad = torch.zeros(ns * N, weight_p.size(1), device=weight_p.device)
    wpad[:weight_p.size(0)] = weight_p.detach()
    return torch.cat([native().pack_weight_f32(wpad[i * N:(i + 1) * N], N, False)[0] for i in range(ns)])


# CSR mode of the fused layer (layer-wise full-neighbourhood inference).  A row with more than CSR_HUB_DEGREE neighbours
# is a hub: a pre-pass sums its adjacency in chunks of CSR_HUB_CHUNK edges (one warp each) and the layer reads the
# chunks' fp32 partial rows instead.  Why 256: a 64-row tile of products-like rows (mean degree ~50) is ~3 500 row reads,
# ~180 per gather warp, and the double-buffered A tile lets one warp fall about one tile's share behind before its CTA
# waits; a 256-neighbour row is ~1.5 shares, while a 3 000-neighbour row would hold the CTA for ~15 tiles.
CSR_HUB_DEGREE = 256
CSR_HUB_CHUNK = 256


class CsrPlan:
    """Static inputs of the CSR mode for one adjacency: row m of a layer aggregates the vids
    ``indices[indptr[m] .. indptr[m + 1])``.  Built once per CSR (hub list, pre-pass chunks, tile-costing degree);
    ``layer`` then runs one layer over all ``n_rows`` rows with no allocation after the first call per width."""

    def __init__(self, indptr: torch.Tensor, indices: torch.Tensor, n_rows: int, hub_degree: int = CSR_HUB_DEGREE):
        dev = indices.device
        n_csr = int(indptr.numel()) - 1
        if n_csr < n_rows:                  # rows without an adjacency row have degree 0
            indptr = torch.cat([indptr, indptr[-1:].expand(n_rows - n_csr)])
        self.indptr = indptr[:n_rows + 1].contiguous()
        self.indices = indices.contiguous()
        deg = self.indptr[1:] - self.indptr[:-1]
        hub = deg > hub_degree
        rows = hub.nonzero().flatten()
        self.n_hub = int(rows.numel())
        light = deg[~hub]
        self.plan_deg = max(1, int(round(float(light.double().mean())))) if light.numel() else 1
        self.n_chunks = 0
        self.hubs = []
        if self.n_hub:
            nch = (deg[rows] + CSR_HUB_CHUNK - 1) // CSR_HUB_CHUNK
            cptr = torch.zeros(self.n_hub + 1, dtype=torch.int64, device=dev)
            cptr[1:] = torch.cumsum(nch, 0)
            self.n_chunks = int(cptr[-1])
            owner = torch.repeat_interleave(torch.arange(self.n_hub, device=dev), nch)
            start = self.indptr[rows][owner] + (torch.arange(self.n_chunks, device=dev) - cptr[owner]) * CSR_HUB_CHUNK
            end = torch.minimum(start + CSR_HUB_CHUNK, self.indptr[rows + 1][owner])
            hub_map = torch.full((n_rows,), -1, dtype=torch.int32, device=dev)
            hub_map[rows] = torch.arange(self.n_hub, dtype=torch.int32, device=dev)
            self.hubs = [hub_map, cptr.to(torch.int32), torch.stack([start, end], 1).contiguous()]
        self._part = {}                     # padded width -> fp32 partial rows of the hub chunks

    def layer(self, tself_desc, tnbr_desc, self_vids: torch.Tensor, out: torch.Tensor, mode: str, w_img: torch.Tensor,
              bias: Optional[torch.Tensor], N: int, n_out: int, relu: bool, out_bf16: bool, n_imgs: int = 1,
              split_k: bool = False):
        """One fused layer over every row: out[m] = act([x_self(self_vids[m]) || agg over the CSR row m] . W^T + b).
        One launch, preceded by the hub pre-pass launch when the CSR has hubs.  ``split_k`` (a split-K layer, see
        ``fused_layer_plan``): a sampled-mode launch with no neighbours first writes x_self . W_self^T into an fp32
        partial, which the CSR launch over the neighbour half adds."""
        C = native()
        hubs = []
        if self.hubs:
            kp = pad_k(int(tnbr_desc[1]))
            if kp not in self._part:
                self._part[kp] = torch.empty(self.n_chunks * kp, dtype=torch.float32, device=self.indices.device)
            hubs = self.hubs + [self._part[kp]]
        part = None
        if split_k:
            M = self_vids.numel()
            part = torch.empty(M, n_imgs * N, dtype=torch.float32, device=self.indices.device)[:, :n_out]
            C.sage_fused_multi(tself_desc, tnbr_desc, [self_vids], [None], [0], [0], [M], [0], [part], [None], MODE[mode],
                               w_img, None, N, n_out, False, False, [], 1, n_imgs, split_half=1)
        C.sage_fused_csr(tself_desc, tnbr_desc, self_vids, self.indptr, self.indices, hubs, out, MODE[mode], w_img, bias, N,
                         n_out, relu, out_bf16, n_imgs, self.plan_deg, 2 if split_k else 0, part)


def logical_weight(weight_p: torch.Tensor, d_self: int, d_nbr: int, mode: str) -> torch.Tensor:
    """[n_out, d_self + d_nbr] (or [n_out, d] for gcn) view of a padded weight."""
    kp_self, _ = padded_dims(d_self, d_nbr, mode)
    if mode == "gcn":
        return weight_p[:, :d_nbr]
    return torch.cat([weight_p[:, :d_self], weight_p[:, kp_self:kp_self + d_nbr]], 1)


def _aligned_rows(x: torch.Tensor) -> torch.Tensor:
    """[n, d] view whose rows start on 16-byte boundaries (the kernel moves 16-byte chunks)."""
    esz = x.element_size()
    if x.stride(1) == 1 and (x.stride(0) * esz) % 16 == 0 and x.data_ptr() % 16 == 0:
        return x
    d = x.size(1)
    per = 16 // esz
    dp = (d + per - 1) // per * per
    buf = torch.zeros(x.size(0), dp, dtype=x.dtype, device=x.device)
    buf[:, :d] = x
    return buf[:, :d]


class _SageFusedFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, weight_p, bias, x_self, x_nbr, tself_desc, self_vids, tnbr_desc, nbr_vids, M, k, mode,
                relu, out_bf16):
        C = native()
        n_out = weight_p.size(0)
        if x_self is not None:
            x_self = _aligned_rows(x_self)
            tself_desc, self_vids = local_table_desc(x_self), None
        if x_nbr is not None:
            x_nbr = _aligned_rows(x_nbr)
            tnbr_desc, nbr_vids = local_table_desc(x_nbr), None
        d_self, d_nbr = int(tself_desc[1]), int(tnbr_desc[1])
        kp_self, kp_nbr = padded_dims(d_self, d_nbr, mode)
        assert weight_p.size(1) == kp_self + kp_nbr, "weight must be in the padded K layout"
        N = pad_n(n_out)
        need_w = ctx.needs_input_grad[0]
        need_x = (x_self is not None and ctx.needs_input_grad[2]) or (x_nbr is not None and ctx.needs_input_grad[3])
        img, w16 = C.pack_weight_f32(weight_p.detach().contiguous(), N, bool(need_x))
        out, a_save = C.sage_fused_forward(tself_desc, self_vids, tnbr_desc, nbr_vids, int(M), int(k), MODE[mode], img,
                                           bias, N, n_out, bool(relu), bool(out_bf16), bool(need_w))
        ctx.save_for_backward(a_save if need_w else None, w16 if need_x else None, out if relu else None)
        ctx.meta = (d_self, d_nbr, kp_self, kp_nbr, int(M), int(k), mode, relu, bias is not None,
                    x_self is not None, x_nbr is not None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        a_save, w16, out = ctx.saved_tensors
        d_self, d_nbr, kp_self, kp_nbr, M, k, mode, relu, has_bias, dense_self, dense_nbr = ctx.meta
        g = grad_out
        if relu:
            g = g * (out > 0).to(g.dtype)
        g16 = g.to(torch.bfloat16)
        dw = db = dxs = dxn = None
        if ctx.needs_input_grad[0]:
            dw = torch.mm(g16.t(), a_save, out_dtype=torch.float32) if _HAS_OUT_DTYPE else (g16.t() @ a_save).float()
        if has_bias and ctx.needs_input_grad[1]:
            db = g.float().sum(0)
        need_xs = dense_self and ctx.needs_input_grad[2]
        need_xn = dense_nbr and ctx.needs_input_grad[3]
        if need_xs or need_xn:
            da = g16 @ w16                                     # [M, K_total]
            if mode == "gcn":
                d_agg = da[:, :d_nbr] * (1.0 / (k + 1))
                if need_xs:
                    dxs = d_agg
                if need_xn:
                    dxn = d_agg[:, None, :].expand(M, k, d_nbr).reshape(M * k, d_nbr)
            else:
                if need_xs:
                    dxs = da[:, :d_self]
                if need_xn:
                    scale = (1.0 / k) if mode == "mean" else 1.0
                    dn = da[:, kp_self:kp_self + d_nbr] * scale
                    dxn = dn[:, None, :].expand(M, k, d_nbr).reshape(M * k, d_nbr)
        return (dw, db, dxs, dxn) + (None,) * 9


# torch.mm(bf16, bf16, out_dtype=fp32) (CUDA only) writes the fp32 gradient without a cast kernel
_HAS_OUT_DTYPE = "out_dtype" in (torch.mm.__doc__ or "")


def pad_weight(weight: torch.Tensor, d_self: int, d_nbr: int, mode: str) -> torch.Tensor:
    """logical [n_out, d_self + d_nbr] (gcn: [n_out, d]) -> padded K layout."""
    kp_self, kp_nbr = padded_dims(d_self, d_nbr, mode)
    wp = torch.zeros(weight.size(0), kp_self + kp_nbr, dtype=weight.dtype, device=weight.device)
    if mode == "gcn":
        wp[:, :d_nbr] = weight
    else:
        wp[:, :d_self] = weight[:, :d_self]
        wp[:, kp_self:kp_self + d_nbr] = weight[:, d_self:]
    return wp


def sage_layer_reference(weight, bias, xs, xn, k, mode="mean", relu=False):
    """Pure torch math on already-gathered rows: xs [M, ds], xn [M*k, dn]; `weight` logical."""
    M = xs.size(0)
    xn3 = xn.view(M, k, -1).float()
    xs = xs.float()
    if mode == "gcn":
        a = (xs + xn3.sum(1)) / (k + 1)
    else:
        agg = xn3.mean(1) if mode == "mean" else xn3.max(1).values if mode == "max" else xn3.sum(1)
        a = torch.cat([xs, agg], 1)
    y = F.linear(a, weight.float(), None if bias is None else bias.float())
    return F.relu(y) if relu else y


def sage_layer(weight_p: torch.Tensor, bias: Optional[torch.Tensor], *, k: int, mode: str = "mean",
               relu: bool = False, out_bf16: bool = False, x_self: Optional[torch.Tensor] = None,
               x_nbr: Optional[torch.Tensor] = None, self_table=None, self_vids: Optional[torch.Tensor] = None,
               nbr_table=None, nbr_vids: Optional[torch.Tensor] = None) -> torch.Tensor:
    """One GraphSAGE layer.  ``weight_p`` is in the padded K layout (see module doc).
    Each of {self, nbr} is either a dense local matrix (``x_*``; gradients flow) or
    (:class:`NodeTable`, vids) read from the sharded store inside the kernel."""
    from . import gather as G
    M = x_self.size(0) if x_self is not None else int(self_vids.numel())
    dev = weight_p.device
    d_self = x_self.size(1) if x_self is not None else self_table.float_dim
    d_nbr = x_nbr.size(1) if x_nbr is not None else nbr_table.float_dim
    use_cuda = dev.type == "cuda" and _config.get().use_peer_kernels
    dt_self = x_self.dtype if x_self is not None else self_table.feats.local.dtype
    dt_nbr = x_nbr.dtype if x_nbr is not None else nbr_table.feats.local.dtype
    kp_s, kp_n = padded_dims(d_self, d_nbr, mode)
    # torch.uint8 = fp8 block-scaled table storage (store/shards.py): only as (table, vids) operands
    ok_dt = (torch.float32, torch.bfloat16) + ((torch.uint8,) if x_self is None and x_nbr is None else ())
    compatible = dt_self == dt_nbr and dt_self in ok_dt and (kp_s == 0 or kp_s == kp_n)
    # max: the fused autograd op's backward spreads the aggregate's gradient like a sum, so max takes the dense path
    if use_cuda and compatible and mode != "max" and fused_supported(d_self, d_nbr, weight_p.size(0), mode, k, dt_self):
        return _SageFusedFn.apply(weight_p, bias, x_self, x_nbr,
                                  None if self_table is None else self_table.feat_desc, self_vids,
                                  None if nbr_table is None else nbr_table.feat_desc, nbr_vids,
                                  M, k, mode, relu, out_bf16)
    # portable / unfused path
    xs = x_self if x_self is not None else G.gather_rows(self_table.rt, self_table.feats, self_table.feat_desc,
                                                         self_vids, d_self)
    xn = x_nbr if x_nbr is not None else G.gather_rows(nbr_table.rt, nbr_table.feats, nbr_table.feat_desc,
                                                       nbr_vids, d_nbr)
    y = sage_layer_reference(logical_weight(weight_p, d_self, d_nbr, mode), bias, xs, xn, k, mode, relu)
    return y.to(torch.bfloat16) if out_bf16 else y
