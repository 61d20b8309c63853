"""K7: dense ``act(x W^T + b)`` on the wgmma tile kernel (``csrc/sage_fused.cu``,
A staged from global memory).  Used by the non-SAGE layers (GAT / GIN / RGCN projections) when
the shapes fit one tile (K <= 512, out <= 256); otherwise - and on CPU - it is ``F.linear``.
Backward = two plain library GEMMs.
Reference counterpart: the dense layers of graphlearn/python/nn/tf/layers/linear_layer.py used by every conv."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn.functional as F

from .. import config as _config
from ..parallel.runtime import native
from . import sage as sage_ops


class _TcLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, relu, out_bf16):
        C = native()
        n_out, k_in = weight.shape
        kp = sage_ops.pad_k(k_in)
        N = sage_ops.pad_n(n_out)
        a = torch.zeros(x.size(0), kp, dtype=torch.bfloat16, device=x.device)
        a[:, :k_in] = x
        wp = torch.zeros(n_out, kp, dtype=torch.float32, device=x.device)
        wp[:, :k_in] = weight
        img, w16 = C.pack_weight_f32(wp, N, True)
        out = C.tc_linear_forward(a, img, bias, N, n_out, bool(relu), bool(out_bf16))
        ctx.save_for_backward(a, w16, out if relu else None)
        ctx.k_in, ctx.relu, ctx.has_bias = k_in, relu, bias is not None
        return out

    @staticmethod
    def backward(ctx, g):
        a, w16, out = ctx.saved_tensors
        if ctx.relu:
            g = g * (out > 0).to(g.dtype)
        g16 = g.to(torch.bfloat16)
        dx = (g16 @ w16)[:, :ctx.k_in] if ctx.needs_input_grad[0] else None
        dw = None
        if ctx.needs_input_grad[1]:
            dw = (torch.mm(g16.t(), a, out_dtype=torch.float32) if sage_ops._HAS_OUT_DTYPE else (g16.t() @ a).float())[:, :ctx.k_in]
        db = g.float().sum(0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        return dx, dw, db, None, None


def tc_linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, relu: bool = False,
              out_bf16: bool = False) -> torch.Tensor:
    k_in, n_out = weight.size(1), weight.size(0)
    fits = k_in <= 512 and n_out <= 256 and sage_ops.smem_fits(sage_ops.pad_k(k_in), sage_ops.pad_n(n_out))
    if x.is_cuda and x.dim() == 2 and _config.get().use_peer_kernels:
        if fits:
            return _TcLinearFn.apply(x, weight, bias, relu, out_bf16)
        if k_in <= 512 and n_out >= 128 and n_out % 2 == 0 and n_out <= 512:
            # W does not fit next to the A tiles: split the output columns (each half is one launch)
            h = n_out // 2
            return torch.cat([tc_linear(x, weight[:h], None if bias is None else bias[:h], relu, out_bf16),
                              tc_linear(x, weight[h:], None if bias is None else bias[h:], relu, out_bf16)], 1)
    y = F.linear(x.float(), weight.float(), None if bias is None else bias.float())
    y = F.relu(y) if relu else y
    return y.to(torch.bfloat16) if out_bf16 else y
