"""Balanced batch dispatch - the capability of the reference's actor engine that survives on GPUs.

The hiactor runtime shards the graph store per core and hands every produced tape to a shard, either round-robin or
ordered by data size so that shards stay evenly loaded (graphlearn/src/actor/runner/tape_dispatcher.cc:61-175,208-218).
On the GPU the SM grid is the sharded executor, but the dispatch problem is still real one level up: seed traversal is
unsharded (every rank walks the nodes IT owns, node_getter.cc:64-92), so ranks see different batch counts and - with
skewed degrees - different amounts of sampling / gather work per batch.  ``gl.enable_actor()`` turns on
:class:`BalancedSeedDispatcher`: at the start of an epoch the ranks exchange their batch weights, a deterministic plan
gives every rank the same number of batches with (greedily) equal total weight, and the seed ids of moved batches travel
in one all-to-all.  No rank idles or truncates its epoch to the shortest shard.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch
import torch.distributed as dist


class TapeDispatcher(object):
    """Pure assignment policies: ``round_robin`` (tape i -> shard i mod n) and ``balanced`` (ordered greedy: every tape
    goes to the currently least-loaded shard, ties to the lowest shard id - tape_dispatcher.cc's data-size-aware mode)."""

    def __init__(self, n_shards: int, strategy: str = "balanced"):
        assert strategy in ("round_robin", "balanced")
        self.n, self.strategy = int(n_shards), strategy

    def assign(self, sizes: Sequence[float]) -> List[int]:
        if self.strategy == "round_robin":
            return [i % self.n for i in range(len(sizes))]
        load = [0.0] * self.n
        count = [0] * self.n
        cap = -(-len(sizes) // self.n)                 # equal batch COUNTS first (collectives run in lock step) ...
        out = []
        for s in sizes:
            cands = [r for r in range(self.n) if count[r] < cap]
            r = min(cands, key=lambda j: (load[j], j))   # ... then equal weight
            load[r] += float(s)
            count[r] += 1
            out.append(r)
        return out


class BalancedSeedDispatcher(object):
    """Epoch-level rebalancing of seed batches across ranks (collective)."""

    def __init__(self, rt, batch_size: int, strategy: str = "balanced"):
        self.rt, self.B, self.strategy = rt, int(batch_size), strategy

    def plan(self, local_seeds: torch.Tensor, weights: Optional[torch.Tensor] = None) -> torch.Tensor:
        """local_seeds: this rank's (already shuffled) seed vids [n]; weights: per-seed work estimate (e.g. out-degree) or
        None.  Returns the seed vids this rank should train on this epoch: whole batches, the same number on every rank."""
        rt, B = self.rt, self.B
        W = rt.world
        n_b = int(local_seeds.numel()) // B
        seeds = local_seeds[:n_b * B].reshape(n_b, B)
        w = (weights[:n_b * B].reshape(n_b, B).sum(1).float() if weights is not None else torch.full((n_b,), float(B))).cpu()
        if W == 1:
            return seeds.reshape(-1)
        all_w = rt.all_gather_object(w.tolist())
        # global tape list in a deterministic order: (rank, local batch index)
        owners = [r for r, ws in enumerate(all_w) for _ in ws]
        sizes = [s for ws in all_w for s in ws]
        total = len(sizes) // W * W                     # whole rounds only: every rank gets len // W batches
        dest = TapeDispatcher(W, self.strategy).assign(sizes[:total])
        # what this rank sends where
        send = [[] for _ in range(W)]
        recv_counts = [0] * W
        idx = 0
        for r, ws in enumerate(all_w):
            for j in range(len(ws)):
                if idx < total:
                    d = dest[idx]
                    if r == rt.rank:
                        send[d].append(j)
                    if d == rt.rank:
                        recv_counts[r] += 1
                idx += 1
        dev = local_seeds.device
        send_t = [seeds[torch.tensor(js, dtype=torch.long, device=dev)].reshape(-1) if js else torch.zeros(0, dtype=torch.int64, device=dev)
                  for js in send]
        recv_t = [torch.zeros(c * B, dtype=torch.int64, device=dev) for c in recv_counts]
        if dev.type == "cuda" and dist.get_backend() == "nccl":
            dist.all_to_all(recv_t, send_t)
        else:
            _gloo_all_to_all(recv_t, send_t, rt)
        return torch.cat(recv_t) if recv_t else torch.zeros(0, dtype=torch.int64, device=dev)


def _gloo_all_to_all(recv_t, send_t, rt):
    """gloo has no all_to_all for uneven splits on every build: exchange through all_gather_object (control-plane sizes)."""
    got = rt.all_gather_object([t.cpu() for t in send_t])
    for r in range(rt.world):
        recv_t[r].copy_(got[r][rt.rank])
