"""EgoGraphSAGE: K layers over a K-hop fixed fan-out ego graph.

Layer i applies the same conv to every adjacent hop pair; K layers consume K
hops (graphlearn/python/nn/tf/model/ego_gnn.py:58-110, ego_layer.py:54-91).
The first layer reads raw features from the sharded store inside the fused
kernel; deeper layers run on dense bf16 activations.

``batch_norm=True`` normalises every hidden layer: each hop tensor of hidden
layer l is ``relu(BN_l(Z))`` with Z the conv output in fp32, ``BN_l`` one
``BatchNorm1d`` (``model.norms[l]``) applied once per hop tensor, the order of
the reference's EgoGNN (graphlearn/python/nn/tf/model/ego_gnn.py:99-104: bn,
then the activation, then dropout).  The hidden convs then have no bias (BN
subtracts the batch mean, and beta is the shift); the top layer keeps its bias.
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn as nn

from ..nn.conv import EgoSAGEConv


class EgoGraphSAGE(nn.Module):
    def __init__(self, in_dim: int, hidden_dim: int, out_dim: int, num_layers: int = 2, agg_type: str = "mean",
                 dropout: float = 0.0, bf16_activations: bool = True, batch_norm: bool = False, bn_eps: float = 1e-5,
                 bn_momentum: float = 0.1):
        super().__init__()
        if batch_norm and not 0.0 < bn_momentum <= 1.0:
            raise ValueError("bn_momentum must be in (0, 1], got %r" % (bn_momentum,))
        dims = [in_dim] + [hidden_dim] * (num_layers - 1) + [out_dim]
        self.convs = nn.ModuleList([EgoSAGEConv(dims[i], dims[i + 1], agg_type, bias=not batch_norm or i == num_layers - 1)
                                    for i in range(num_layers)])
        self.num_layers = num_layers
        self.dropout = dropout
        self.bf16 = bf16_activations
        self.batch_norm = bool(batch_norm)
        if batch_norm:
            self.norms = nn.ModuleList([nn.BatchNorm1d(hidden_dim, eps=bn_eps, momentum=bn_momentum)
                                        for _ in range(num_layers - 1)])

    def _act(self, l: int, z: torch.Tensor) -> torch.Tensor:
        """hidden layer l's output from its fp32 conv output z (batch norm only): relu(BN_l(z)), bf16 when the model
        keeps bf16 activations"""
        h = torch.relu(self.norms[l](z))
        return h.to(torch.bfloat16) if self.bf16 else h

    def _conv(self, l: int, x, nbr, k: int, last: bool):
        if self.batch_norm and not last:
            return self._act(l, self.convs[l](x, nbr, k, relu=False, out_bf16=False))
        return self.convs[l](x, nbr, k, relu=not last, out_bf16=self.bf16 and not last)

    def forward_store(self, table, hops: Sequence[torch.Tensor], fanouts: Sequence[int]) -> torch.Tensor:
        """hops[0] = seed vids [B]; hops[i] = vids [B*k1*..*k_i]; returns logits [B, out]."""
        L = self.num_layers
        assert len(hops) == L + 1 and len(fanouts) == L
        h: List[torch.Tensor] = []
        last = L == 1
        for i in range(L):      # layer 0 straight from the store
            if self.batch_norm and not last:
                h.append(self._act(0, self.convs[0].forward_store(table, hops[i], hops[i + 1], fanouts[i])))
            else:
                h.append(self.convs[0].forward_store(table, hops[i], hops[i + 1], fanouts[i], relu=not last,
                                                     out_bf16=self.bf16 and not last))
        for l in range(1, L):
            last = l == L - 1
            nh = []
            for i in range(L - l):
                x = h[i]
                if self.training and self.dropout > 0:
                    x = torch.nn.functional.dropout(x, self.dropout)
                nh.append(self._conv(l, x, h[i + 1], fanouts[i], last))
            h = nh
        return h[0].float()

    def forward(self, xs: Sequence[torch.Tensor], fanouts: Sequence[int]) -> torch.Tensor:
        """Dense variant: xs[i] = features of hop i ([B*prod(k), d])."""
        L = self.num_layers
        h = list(xs)
        for l in range(L):
            last = l == L - 1
            h = [self._conv(l, h[i], h[i + 1], fanouts[i], last) for i in range(L - l)]
        return h[0].float()
