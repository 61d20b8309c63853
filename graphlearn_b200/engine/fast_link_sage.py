"""Hand-scheduled training step for unsupervised (link-prediction) EgoGraphSAGE.

The objective of graphlearn/examples/tf/ego_sage/train_unsupervised.py: the roots of a step are B positive edges
(src, dst) plus ``neg_num`` negatives drawn per src, ONE shared encoder embeds the ego graphs of all of them, and the
loss is a dot-product loss over the top-layer embeddings (``nn/loss.py``: ``sigmoid_cross_entropy_loss`` or
``unsupervised_softmax_cross_entropy_loss``).

It is ``FastSageTrainer`` with R = B * (2 + neg_num) roots in the order [src | dst | negatives of src 0 | ...]: hop
buffers, layers, backward and the fused Adam kernel are the supervised engine's.  Only the roots and the top-layer
loss differ:

  sampling branch   link_roots (staged edge batch -> src / dst roots)          [when staged from the host]
                    negative_sample_kernel -> roots[2B:] (draw + neighbour rejection, written in place)
                    sample hops 1..L over all R roots, advance the counters
  top layer         fp32 embeddings, no ReLU, never fused with a loss; link_loss_kernel writes the loss, the gradient
                    of every root's embedding and the top bias gradient

Multi-GPU: every rank traverses its own edges (src is local); dst and negatives may be remote and are read through
the peer tables like any other hop; gradients are averaged in ``adam_pack``.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import config as _config
from ..ops.negative import _WeightedSampler, _shard_offsets
from .fast_sage import FastSageTrainer

LOSS_KINDS = {"sigmoid": 0, "softmax": 1}


class FastLinkSageTrainer(FastSageTrainer):
    _fuse_ce = False
    NEG_SALT = 0x4E4547          # RNG salt of the negative draws; the hop draws use the salts 1..L

    def __init__(self, rt, nodes, csr, model, fanouts, batch_size: int, neg_num: int, neg_strategy: str = "random",
                 loss: str = "sigmoid", temperature: float = 1.0, lr: float = 3e-3, use_cuda_graph: bool = True,
                 allreduce: str = "peer", seed: int = 0, **kw):
        if loss not in LOSS_KINDS:
            raise ValueError("loss must be 'sigmoid' or 'softmax', got %r" % (loss,))
        if neg_strategy not in ("random", "in_degree"):
            raise ValueError("neg_strategy must be 'random' or 'in_degree', got %r" % (neg_strategy,))
        if csr.src_type != csr.dst_type or csr.dst_type != nodes.type:
            raise ValueError("link training needs a homogeneous edge type whose src and dst are the encoder's node type")
        if int(batch_size) < 1 or int(neg_num) < 1:
            raise ValueError("batch_size and neg_num must be positive")
        if model.convs[-1].out_dim > 256:
            raise ValueError("link training supports embeddings up to 256 wide")
        if temperature <= 0:
            raise ValueError("temperature must be positive")
        self.batch_size = int(batch_size)            # positive edges per step
        self.neg_num = int(neg_num)
        self.neg_strategy = neg_strategy
        self.loss_kind = loss
        self.temperature = float(temperature)
        super().__init__(rt, nodes, csr, model, fanouts, self.batch_size * (2 + self.neg_num), lr=lr,
                         use_cuda_graph=use_cuda_graph, allreduce=allreduce, seed=seed, **kw)
        dev = rt.device
        # negative draws: the kernel branch of ops/negative.py::edge_negative (same universe, CDF and retries)
        self._neg_off, self._neg_total = _shard_offsets(nodes, dev)
        self._neg_cum = None
        if neg_strategy == "in_degree":
            self._neg_cum = _WeightedSampler(rt, self._local_in_degrees()).cum
        self._neg_retry = int(_config.get().neg_sampling_retry_times)
        self._edge_rows = csr._row_of_edge
        self._edge_dst = csr.indices.local

    def _local_in_degrees(self) -> torch.Tensor:
        """in-degree of every node this rank owns under the edge type (what ``GraphStore.reverse_csr`` counts)"""
        W, nodes = self.rt.world, self.nodes
        dst = self.csr.indices.local
        dst = dst[dst >= 0]
        if W == 1:
            return torch.bincount(dst, minlength=nodes.n_local)[:nodes.n_local].float()
        import torch.distributed as dist
        n_vid = max(int(n) for n in nodes.nrows) * W
        cnt = torch.bincount(dst, minlength=n_vid)[:n_vid]
        dist.all_reduce(cnt)
        return cnt[self.rt.rank::W][:nodes.n_local].float()

    # ------------------------------------------------------------------ front end
    @classmethod
    def from_graph(cls, graph, edge_type: str, model, fanouts, batch_size: int, neg_num: int,
                   **kw) -> "FastLinkSageTrainer":
        """Train on the edges of ``edge_type`` of a ``gl.Graph`` (src type == dst type), the reference's
        ``E(edge_type).batch(B).shuffle(traverse=True)`` + ``outNeg(edge_type).sample(neg_num)`` + ego graphs of
        src, dst and negatives over ``outV(edge_type)`` hops.  Drive it with ``step_edges()``."""
        store = graph.store
        if edge_type not in store.edges:
            raise KeyError("unknown edge type %r" % (edge_type,))
        csr = store.edges[edge_type]
        if csr.src_type != csr.dst_type:
            raise ValueError("link training needs src type == dst type (%r -> %r)" % (csr.src_type, csr.dst_type))
        if kw.get("strategy") == "in_degree":
            store.ensure_indegree_weights(edge_type)
        tr = cls(graph.runtime, store.nodes[csr.src_type], csr, model, fanouts, batch_size, neg_num, **kw)
        tr.graph_api = graph
        return tr

    # ------------------------------------------------------------------ roots and loss of the shared step
    def _stage(self, roots: torch.Tensor, host_slot: int):
        self.C.link_roots(roots, self._h_seeds_dev[host_slot][:2 * self.batch_size + 1], self._edge_rows,
                          self._edge_dst, self.rt.world, self.rt.rank)

    def _draw_roots(self, roots: torch.Tensor):
        B = self.batch_size
        self.C.negative_sample(self.csr.desc, roots[:B], self.neg_num, self._neg_cum, self._neg_off, self._neg_total,
                               self.neg_strategy == "in_degree", self._neg_retry, 1024, self.rng.state, self.NEG_SALT,
                               roots[2 * B:])

    def _top_loss(self, seeds: torch.Tensor):
        top = self.layers[-1]
        self.C.link_loss(top.H, self.batch_size, self.neg_num, LOSS_KINDS[self.loss_kind], self.temperature,
                         self.loss, top.dZ, top.db)

    def _fill_slot(self, slot: int, first: torch.Tensor, dst: Optional[torch.Tensor] = None):
        """pinned staging slot: [0, B) src vids or CSR positions, [B, 2B) dst vids, [2B] what [0, B) holds"""
        B = self.batch_size
        if first.numel() != B or (dst is not None and dst.numel() != B):
            raise ValueError("a step takes exactly batch_size = %d edges" % B)
        h = self._h_seeds2[slot]
        h[:B].copy_(first.reshape(-1))
        if dst is None:
            h[2 * B] = 1
        else:
            h[B:2 * B].copy_(dst.reshape(-1))
            h[2 * B] = 0

    def _put_roots(self, roots: torch.Tensor, src: torch.Tensor, dst: torch.Tensor):
        B = self.batch_size
        self.C.copy_i64(roots[:B], src)
        self.C.copy_i64(roots[B:2 * B], dst)

    # ------------------------------------------------------------------ public steps
    def step(self, src_ids_host: torch.Tensor, dst_ids_host: torch.Tensor) -> torch.Tensor:
        """End-to-end step on B host edges (src / dst vids).  Asynchronous, and with CUDA graphs pipelined exactly like
        ``FastSageTrainer.step``: the call stages its edges and trains on those of the previous call; the returned
        pinned tensor receives that step's loss."""
        return self._step_staged(src_ids_host, dst_ids_host)

    def step_edges(self) -> torch.Tensor:
        """One step on the next B local edges of the edge traversal ``E(t).batch(B).shuffle(traverse=True)``: every
        local edge once per epoch, full batches only; raises ``OutOfRangeError`` at the end of an epoch."""
        if self._q_iter is None:        # the traversal hands CSR positions to ``_fill_slot``
            self._set_traversal(self.csr.insertion_pos().cpu(), self.batch_size, "shuffle")
        return self.step_query()

    def step_device(self, next_src: Optional[torch.Tensor] = None, next_dst: Optional[torch.Tensor] = None):
        """Device-only step.  ``next_src`` / ``next_dst`` (device int64 [B] vids) are the edges of the batch the replay
        samples for the FOLLOWING step; without them the resident edges get fresh negatives and hops."""
        self._step_device(next_src, next_dst)

    @torch.no_grad()
    def embed(self, vids: torch.Tensor) -> torch.Tensor:
        """fp32 embeddings of `vids` (device int64) from the trained encoder (``forward_store`` on fresh hops)."""
        return self.predict(vids)
