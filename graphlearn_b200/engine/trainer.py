"""Sampled-subgraph training step engine.

One ``step`` = sample K hops -> fused gather/aggregate/GEMM forward -> loss ->
backward -> (multi-GPU) peer-memory gradient all-reduce -> fused Adam.  The
whole step is a stream-ordered chain of device work with static shapes (fixed
fan-out + padding), so it is captured once into a CUDA graph and replayed:
this is the GPU replacement for the reference's sampling||training
producer/consumer pipeline (DagScheduler -> TapeStore -> Dataset prefetch,
graphlearn/src/core/runner/dag_scheduler.cc:45-86, dag/tape.cc:110-153) -
there is no host in the loop to overlap with any more.

The only per-step host->device traffic is the seed-id batch (pinned host
buffer -> device) and the only device->host traffic is the loss scalar.
"""
from __future__ import annotations

from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from ..ops import comm as comm_ops
from ..ops import gather as G
from ..ops import rng as rng_ops
from ..ops import sampling as S
from ..parallel.runtime import Runtime
from ..store.shards import CsrShard, NodeTable


class SageTrainer:
    def __init__(self, rt: Runtime, nodes: NodeTable, csr: CsrShard, model: torch.nn.Module,
                 fanouts: Sequence[int], batch_size: int, lr: float = 3e-3, strategy: str = "random",
                 use_cuda_graph: bool = True, allreduce: str = "peer", seed: int = 0):
        self.rt, self.nodes, self.csr, self.model = rt, nodes, csr, model
        self.fanouts = list(fanouts)
        self.B = int(batch_size)
        self.strategy = strategy
        self.rng = rng_ops.DeviceRng(rt, seed)
        self.flat_p, self.flat_g = comm_ops.flatten_module(model)
        if rt.world > 1:            # replicas start from rank 0's initialisation (what DDP does at construction)
            import torch.distributed as dist
            with torch.no_grad():
                dist.broadcast(self.flat_p, src=0)
        self.opt = comm_ops.FlatAdam(self.flat_p, self.flat_g, lr=lr)
        self.ar = comm_ops.PeerAllReduce(rt, self.flat_g.numel(), backend=allreduce)
        self.seeds = torch.zeros(self.B, dtype=torch.int64, device=rt.device)     # static input buffer
        self.loss = torch.zeros((), dtype=torch.float32, device=rt.device)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.use_graph = bool(use_cuda_graph and rt.is_cuda)
        self._steps = 0
        self.kernel_launches_per_step = None
        if rt.is_cuda:
            self.h_seeds = torch.zeros(self.B, dtype=torch.int64).pin_memory()
            self.h_loss = torch.zeros((), dtype=torch.float32).pin_memory()
        else:
            self.h_seeds = torch.zeros(self.B, dtype=torch.int64)
            self.h_loss = torch.zeros((), dtype=torch.float32)

    # ------------------------------------------------------------------ one step of device work
    def sample(self, seeds: torch.Tensor):
        hops = [seeds]
        cur = seeds
        for i, k in enumerate(self.fanouts):
            nbr, _ = S.sample_neighbors(self.csr, cur, k, self.strategy, want_eids=False, rng=self.rng, salt=i + 1)
            cur = nbr.reshape(-1)
            hops.append(cur)
        return hops

    def _step_body(self):
        self.flat_g.zero_()
        hops = self.sample(self.seeds)
        logits = self.model.forward_store(self.nodes, hops, self.fanouts)
        # seeds are always owned by this rank (every rank traverses its own shard, like the
        # reference's unsharded GetNodes) -> labels are a local lookup
        labels = self.nodes.labels.local[torch.div(self.seeds, self.rt.world, rounding_mode="floor")]
        loss = F.cross_entropy(logits, labels)
        loss.backward()
        self.ar(self.flat_g, average=True)
        self.opt.step(self.rng.state)           # also advances the sampling RNG offset
        self.loss.copy_(loss.detach())

    def capture(self, warmup: int = 3):
        """Warm up eagerly on a side stream, then capture the step into a CUDA graph."""
        if not self.use_graph or self.graph is not None:
            return
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                self._step_body()
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.rt.barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._step_body()
        self.graph = g
        torch.cuda.synchronize()
        self.rt.barrier()

    def step_device(self):
        """Device-only step on the current contents of ``self.seeds``."""
        if self.graph is not None:
            self.graph.replay()
        else:
            self._step_body()
        self._steps += 1

    def step(self, seed_ids_host: torch.Tensor) -> torch.Tensor:
        """End-to-end step through the public path: pinned-host seed ids -> device,
        train, loss -> pinned host (async; synchronise before reading)."""
        self.h_seeds.copy_(seed_ids_host)
        self.seeds.copy_(self.h_seeds, non_blocking=True)
        self.step_device()
        self.h_loss.copy_(self.loss, non_blocking=True)
        return self.h_loss

    # ------------------------------------------------------------------ checkpoint
    def state_dict(self):
        return {"model": self.flat_p.clone(), "opt": self.opt.state_dict(), "rng": self.rng.state_dict(),
                "steps": self._steps}

    def load_state_dict(self, sd):
        self.flat_p.copy_(sd["model"])
        self.opt.load_state_dict(sd["opt"])
        self.rng.load_state_dict(sd["rng"])
        self._steps = int(sd["steps"])
