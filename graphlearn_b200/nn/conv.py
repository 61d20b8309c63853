"""GNN layers on EgoGraphs (dense, fixed fan-out) - PyTorch modules.

Re-implements the math of the reference's TF1 layers
(graphlearn/python/nn/tf/layers/ego_{sage,gat,gin,rgcn}_conv.py, SURVEY 2.8)
with the SAGE layer running on the fused sm_90a kernel.
"""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import sage as sage_ops


class EgoSAGEConv(nn.Module):
    """out = W . [x || agg(nbrs)]  (agg in mean|sum|max) or 'gcn' = W . mean({x} U nbrs).

    ego_sage_conv.py:71-106.  ``forward`` takes already-gathered dense tensors;
    ``forward_store`` reads rows straight from the sharded feature store inside
    the fused kernel (no [B*k, D] intermediate)."""

    def __init__(self, in_dim, out_dim, agg_type="mean", bias=True, in_nbr_dim=None):
        super().__init__()
        self.in_self = int(in_dim if not isinstance(in_dim, (tuple, list)) else in_dim[0])
        self.in_nbr = int(in_nbr_dim if in_nbr_dim is not None else
                          (in_dim[1] if isinstance(in_dim, (tuple, list)) else in_dim))
        self.out_dim = int(out_dim)
        self.agg_type = agg_type
        assert agg_type in ("mean", "sum", "max", "gcn")
        k_in = self.in_nbr if agg_type == "gcn" else self.in_self + self.in_nbr
        self._mode = "mean" if agg_type == "max" else agg_type
        w = torch.empty(out_dim, k_in)
        nn.init.kaiming_uniform_(w, a=math.sqrt(5))
        # stored in the fused kernel's padded K layout (pad columns are zero and stay zero)
        self.weight_p = nn.Parameter(sage_ops.pad_weight(w, self.in_self, self.in_nbr, self._mode))
        self.bias = nn.Parameter(torch.zeros(out_dim)) if bias else None

    @property
    def weight(self):
        """Logical [out, in_self + in_nbr] weight (gcn: [out, in])."""
        return sage_ops.logical_weight(self.weight_p, self.in_self, self.in_nbr, self._mode)

    def forward(self, x, neighbor, expand, relu=False, out_bf16=False):
        """x [M, d], neighbor [M*k, d_n], expand = k."""
        if self.agg_type == "max":
            agg = neighbor.view(-1, expand, neighbor.size(-1)).float().max(1).values
            y = F.linear(torch.cat([x.float(), agg], 1), self.weight, self.bias)
            y = F.relu(y) if relu else y
            return y.to(torch.bfloat16) if out_bf16 else y
        return sage_ops.sage_layer(self.weight_p, self.bias, k=expand, mode=self.agg_type, relu=relu,
                                   out_bf16=out_bf16, x_self=x, x_nbr=neighbor)

    def forward_store(self, table, self_vids, nbr_vids, expand, relu=False, out_bf16=False, nbr_table=None):
        if self.agg_type == "max":
            from ..ops import gather as G
            nt = nbr_table or table
            xs = G.gather_rows(table.rt, table.feats, table.feat_desc, self_vids, table.float_dim)
            xn = G.gather_rows(nt.rt, nt.feats, nt.feat_desc, nbr_vids, nt.float_dim)
            return self.forward(xs, xn, expand, relu, out_bf16)
        return sage_ops.sage_layer(self.weight_p, self.bias, k=expand, mode=self.agg_type, relu=relu,
                                   out_bf16=out_bf16, self_table=table, self_vids=self_vids.reshape(-1),
                                   nbr_table=nbr_table or table, nbr_vids=nbr_vids.reshape(-1))


class EgoGATConv(nn.Module):
    """Multi-head attention over a fixed fan-out neighbourhood - math and parameters of the reference
    (ego_gat_conv.py:50-117): per head  x' = W_x x (+b),  n' = W_n n (+b),  e = LeakyReLU(att . [x' || n'] (+b)),
    coef = softmax over the k NEIGHBOURS, ret = sum_j coef_j n'_j; heads are AVERAGED.  ``W_n`` is ``W_x`` when
    both sides have the same input dimension (``in_dim`` an int), like the reference; ``use_bias`` (default False,
    like the reference) adds biases to all three linear maps.

    Execution: the attention logit is linear in the raw rows, so the layer runs as ONE gather + online-softmax
    kernel that aggregates RAW rows per head (``ops.gat``) followed by ONE tensor-core GEMM with the concatenated
    ``W_n`` - no [M*k, H*D] projected neighbour tensor."""

    def __init__(self, in_dim, out_dim, num_head=1, use_bias=False, attn_drop=0.0, negative_slope=0.2, bias=None):
        super().__init__()
        homo = not isinstance(in_dim, (tuple, list))
        self.in_self = int(in_dim if homo else in_dim[0])
        self.in_nbr = int(in_dim if homo else in_dim[1])
        self.out_dim, self.num_head = int(out_dim), int(num_head)
        use_bias = bool(use_bias if bias is None else bias)          # `bias=` kept as an alias of use_bias
        H, D = self.num_head, self.out_dim
        self.lin_self = nn.Linear(self.in_self, D * H, bias=use_bias)
        self.lin_nbr = self.lin_self if homo else nn.Linear(self.in_nbr, D * H, bias=use_bias)
        self.att = nn.Parameter(torch.empty(H, 2 * D))                # [a_x || a_n] per head
        self.att_bias = nn.Parameter(torch.zeros(H)) if use_bias else None
        self.attn_drop, self.slope = attn_drop, negative_slope
        nn.init.xavier_uniform_(self.att)

    # ---- the two equivalent evaluations
    def _logit_vectors(self):
        """u_x [H, d_self], u_n [H, d_nbr], c [H] with e = LeakyReLU(u_x . x + u_n . n + c)."""
        H, D = self.num_head, self.out_dim
        a_x, a_n = self.att[:, :D], self.att[:, D:]
        wx = self.lin_self.weight.view(H, D, self.in_self)
        wn = self.lin_nbr.weight.view(H, D, self.in_nbr)
        u_x = torch.einsum("hd,hdi->hi", a_x, wx)
        u_n = torch.einsum("hd,hdi->hi", a_n, wn)
        c = torch.zeros(H, device=self.att.device)
        if self.lin_self.bias is not None:
            c = c + (a_x * self.lin_self.bias.view(H, D)).sum(1)
        if self.lin_nbr.bias is not None:
            c = c + (a_n * self.lin_nbr.bias.view(H, D)).sum(1)
        if self.att_bias is not None:
            c = c + self.att_bias
        return u_x, u_n, c

    def forward_reference(self, x, neighbor, expand):
        """Literal transcription of the reference layer (projects every neighbour row first) - the parity oracle."""
        M, H, D = x.size(0), self.num_head, self.out_dim
        xs = self.lin_self(x.float()).view(M, 1, H, D)
        xn = self.lin_nbr(neighbor.float()).view(M, expand, H, D)
        a_x, a_n = self.att[:, :D], self.att[:, D:]
        score = (xs * a_x).sum(-1) + (xn * a_n).sum(-1)                       # [M, k, H]
        if self.att_bias is not None:
            score = score + self.att_bias
        coef = torch.softmax(F.leaky_relu(score, self.slope), dim=1)          # over the k neighbours only
        if self.training and self.attn_drop > 0:
            coef = F.dropout(coef, self.attn_drop)
        return (coef.unsqueeze(-1) * xn).sum(1).mean(1)                       # average heads

    def _project(self, agg):
        """out = mean_h ( W_n,h agg_h + b_n,h ) as one GEMM over the concatenated, kp-padded per-head blocks."""
        from ..ops.linear import tc_linear
        H, D = self.num_head, self.out_dim
        kp = agg.size(1) // H
        wn = self.lin_nbr.weight.view(H, D, self.in_nbr)
        wcat = torch.cat([F.pad(wn[h], (0, kp - self.in_nbr)) for h in range(H)], 1) / H          # [D, H * kp]
        b = self.lin_nbr.bias.view(H, D).mean(0) if self.lin_nbr.bias is not None else None
        return tc_linear(agg, wcat, b)

    def forward(self, x, neighbor, expand):
        if self.training and self.attn_drop > 0:
            return self.forward_reference(x, neighbor, expand)               # dropout on the coefficients: literal path
        from ..ops import gat as gat_ops
        u_x, u_n, c = self._logit_vectors()
        agg = gat_ops.gat_aggregate(u_x, u_n, c, k=expand, slope=self.slope, x_self=x, x_nbr=neighbor)
        return self._project(agg).float()

    def forward_store(self, table, self_vids, nbr_vids, expand, nbr_table=None):
        """First layer: rows are pulled from the sharded feature store inside the attention kernel."""
        from ..ops import gat as gat_ops
        u_x, u_n, c = self._logit_vectors()
        agg = gat_ops.gat_aggregate(u_x, u_n, c, k=expand, slope=self.slope, self_table=table, self_vids=self_vids,
                                    nbr_table=nbr_table or table, nbr_vids=nbr_vids)
        return self._project(agg).float()


class EgoGINConv(nn.Module):
    """W((1 + eps) x + sum(nbrs))  (ego_gin_conv.py:80-100); separate input projections when the
    self / neighbour dims differ."""

    def __init__(self, in_dim, out_dim, eps=0.0, train_eps=False, bias=True):
        super().__init__()
        self.in_self = int(in_dim if not isinstance(in_dim, (tuple, list)) else in_dim[0])
        self.in_nbr = int(in_dim if not isinstance(in_dim, (tuple, list)) else in_dim[1])
        self.eps = nn.Parameter(torch.tensor(float(eps))) if train_eps else float(eps)
        self.proj_self = self.proj_nbr = None
        if self.in_self != self.in_nbr:
            self.proj_self = nn.Linear(self.in_self, out_dim, bias=False)
            self.proj_nbr = nn.Linear(self.in_nbr, out_dim, bias=False)
            self.lin = nn.Linear(out_dim, out_dim, bias=bias)
        else:
            self.lin = nn.Linear(self.in_self, out_dim, bias=bias)

    def forward(self, x, neighbor, expand):
        agg = neighbor.float().view(x.size(0), expand, -1).sum(1)
        xs = x.float()
        if self.proj_self is not None:
            xs, agg = self.proj_self(xs), self.proj_nbr(agg)
        return self.lin((1.0 + self.eps) * xs + agg)


class EgoRGCNConv(nn.Module):
    """Relational GCN on ego graphs: sum_r mean_r(nbrs_r) W_r + x W_0 with basis or block-diagonal
    weight decomposition (ego_rgcn_conv.py:108-139)."""

    def __init__(self, in_dim, out_dim, num_relations, num_bases=None, num_blocks=None, bias=True):
        super().__init__()
        self.in_dim, self.out_dim, self.R = int(in_dim), int(out_dim), int(num_relations)
        self.num_bases, self.num_blocks = num_bases, num_blocks
        if num_bases:
            self.basis = nn.Parameter(torch.empty(num_bases, in_dim, out_dim))
            self.comp = nn.Parameter(torch.empty(num_relations, num_bases))
            nn.init.xavier_uniform_(self.basis)
            nn.init.xavier_uniform_(self.comp)
        elif num_blocks:
            assert in_dim % num_blocks == 0 and out_dim % num_blocks == 0
            self.blocks = nn.Parameter(torch.empty(num_relations, num_blocks, in_dim // num_blocks, out_dim // num_blocks))
            nn.init.xavier_uniform_(self.blocks)
        else:
            self.weight = nn.Parameter(torch.empty(num_relations, in_dim, out_dim))
            nn.init.xavier_uniform_(self.weight)
        self.root = nn.Linear(in_dim, out_dim, bias=bias)

    def relation_weights(self):
        if self.num_bases:
            return torch.einsum("rb,bio->rio", self.comp, self.basis)
        if self.num_blocks:
            return torch.stack([torch.block_diag(*self.blocks[r]) for r in range(self.R)])
        return self.weight

    def forward(self, x, neighbors, expands):
        """neighbors: list (one per relation) of [M*k_r, d]; expands: list of k_r."""
        W = self.relation_weights()
        out = self.root(x.float())
        for r, (nb, k) in enumerate(zip(neighbors, expands)):
            out = out + nb.float().view(x.size(0), k, -1).mean(1) @ W[r]
        return out


class EgoLayer(nn.Module):
    """Applies one conv to every adjacent hop pair (ego_layer.py:54-91)."""

    def __init__(self, convs):
        super().__init__()
        self.convs = nn.ModuleList(convs)

    def append(self, conv):
        """add the conv of one more hop pair (ego_layer.py:94-95)"""
        self.convs.append(conv)
        return self

    def forward(self, x_list, expands):
        assert len(self.convs) == len(x_list) - 1
        return [self.convs[i](x_list[i], x_list[i + 1], expands[i]) for i in range(len(x_list) - 1)]


class TimeEncoder(nn.Module):
    """Functional time encoding cos(t * w + b) used by the temporal models (EgoTGAT / TGN:
    graphlearn/python/nn/tf/data/temporal_graph.py, examples/tf/ego_tgat)."""

    def __init__(self, dim: int):
        super().__init__()
        self.lin = nn.Linear(1, dim)
        with torch.no_grad():
            self.lin.weight.copy_((1.0 / 10 ** torch.linspace(0, 9, dim)).view(dim, 1))
            self.lin.bias.zero_()

    def forward(self, t: torch.Tensor) -> torch.Tensor:
        return torch.cos(self.lin(t.float().unsqueeze(-1)))


class EgoTGATConv(nn.Module):
    """Temporal GAT layer on ego graphs: attention over the k most recent neighbours with
    [feature || time-encoding(t_self - t_edge)] keys (ego_tgat)."""

    def __init__(self, in_dim: int, out_dim: int, time_dim: int = 16, num_head: int = 2):
        super().__init__()
        self.time = TimeEncoder(time_dim)
        self.att = EgoGATConv((in_dim + time_dim, in_dim + time_dim), out_dim, num_head)

    def forward(self, x, neighbor, expand, t_self, t_edge):
        """x [M,d], neighbor [M*k,d], t_self [M], t_edge [M*k]."""
        dt = t_self.repeat_interleave(expand) - t_edge
        xs = torch.cat([x.float(), self.time(torch.zeros_like(t_self))], 1)
        xn = torch.cat([neighbor.float(), self.time(dt)], 1)
        return self.att(xs, xn, expand)


class EgoConv(nn.Module):
    """Abstract EgoGraph convolution (ego_layer.py:25-39): ``forward(x [n, d_x], neighbor [n * expand, d_n], expand)`` ->
    [n, out].  ``EgoSAGEConv / EgoGATConv / EgoGINConv / EgoRGCNConv`` follow this contract; subclass it for custom layers
    that ``EgoLayer`` can stack."""

    def forward(self, x, neighbor, expand):
        raise NotImplementedError


class SubConv(nn.Module):
    """Abstract SubGraph convolution (sub_conv.py:25-37): ``forward(edge_index [2, m], node_vec [n, d])`` -> [n, out]
    (``GCNConv / SAGEConv / GATConv`` in ``nn.sparse_conv`` take ``(x, edge_index)``; ``HeteroConv`` accepts both orders)."""

    def forward(self, edge_index, node_vec, **kwargs):
        raise NotImplementedError


class LinearLayer(nn.Module):
    """``y = act(x W + b)`` with lazily inferred input width (linear_layer.py:29-75: ``LinearLayer(name, input_dim,
    output_dim, use_bias)``)."""

    def __init__(self, name="linear", input_dim=None, output_dim=1, use_bias=True, activation=None):
        super().__init__()
        self.name = name
        self.lin = nn.Linear(int(input_dim), int(output_dim), bias=use_bias) if input_dim else nn.LazyLinear(int(output_dim), bias=use_bias)
        self.activation = activation

    def forward(self, x):
        y = self.lin(x)
        return self.activation(y) if self.activation is not None else y
