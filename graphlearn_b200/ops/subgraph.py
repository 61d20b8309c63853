"""Induced-subgraph sampling and relabelling (K4).

Semantics (graphlearn/src/core/operator/subgraph/subgraph_sampler.cc:35-95):
seeds are optionally expanded hop by hop, the union of nodes is de-duplicated,
every node's (capped) full neighbourhood is intersected with the node set and
each hit is emitted in BOTH directions as (row, col, edge id); with
``need_dist`` the SEAL double-radius labels are BFS distances to src (node 0)
with dst removed and to dst (node 1) with src removed.

GPU design: rows come from the peer-memory full sampler; the intersection is
a sort + ``searchsorted`` membership test on the device (sorted-set intersect)
instead of per-row hash maps; BFS is frontier expansion with index ops.
"""
from __future__ import annotations

from typing import List, Optional

import torch

from .. import config as _config
from . import sampling as S


def unique_relabel(ids: torch.Tensor):
    """unique ids in first-occurrence order + compact index of every input id (K4 dedup/relabel; device hash
    table on CUDA, ops/sparse.py:Relabel)."""
    from .sparse import Relabel
    r = Relabel(ids)
    return r.uniq, r.inverse


def _bfs(n: int, row: torch.Tensor, col: torch.Tensor, start: int, removed: int, max_iters: int = 64):
    dev = row.device
    INF = 2 ** 31 - 1
    dist = torch.full((n,), INF, dtype=torch.int64, device=dev)
    if n == 0:
        return dist
    keep = (row != removed) & (col != removed)
    r, c = row[keep], col[keep]
    dist[start] = 0
    frontier = torch.zeros(n, dtype=torch.bool, device=dev)
    frontier[start] = True
    for d in range(1, max_iters):
        nxt = torch.zeros(n, dtype=torch.bool, device=dev)
        nxt[c[frontier[r]]] = True
        nxt &= dist == INF
        if not bool(nxt.any()):
            break
        dist[nxt] = d
        frontier = nxt
    return dist


def induce_subgraph(store, etype: str, seeds: torch.Tensor, num_nbrs: List[int], need_dist: bool = False,
                    src: Optional[torch.Tensor] = None, dst: Optional[torch.Tensor] = None, rng=None):
    cfg = _config.get()
    csr = store.edges[etype]
    dev = seeds.device
    frontier = seeds.reshape(-1)
    all_nodes = [frontier]
    for hop, k in enumerate(num_nbrs):
        nbr, _ = S.sample_neighbors(csr, frontier, int(k), "random", want_eids=False, rng=rng, salt=900 + hop)
        frontier = nbr.reshape(-1)
        all_nodes.append(frontier)
    cat = torch.cat(all_nodes)
    cat = cat[cat >= 0]
    from .sparse import Relabel
    if need_dist and src is not None and dst is not None and src.numel() == 1:
        # SEAL: src is node 0, dst is node 1 (first-occurrence order puts them first)
        cat = torch.cat([src.reshape(-1)[:1], dst.reshape(-1)[:1], cat])
    rl = Relabel(cat)          # K4: device hash table, unique ids in first-occurrence order (seeds first)
    nodes = rl.uniq
    n = int(nodes.numel())
    vals, eids, offs = S.sample_full(csr, nodes, cap=cfg.default_full_nbr_num, want_eids=True)
    counts = offs[1:] - offs[:-1]
    rows = torch.repeat_interleave(torch.arange(n, device=dev), counts)
    cidx = rl.lookup(vals)     # membership test + local index in one table probe
    hit = cidx >= 0
    r, c, e = rows[hit], cidx[hit], eids[hit]
    # the reference's order (subgraph_sampler.cc / its python checks): stored edges by (row index, col index), each followed
    # by its mirrored entry
    order = torch.argsort(r * max(n, 1) + c, stable=True)
    r, c, e = r[order], c[order], e[order]
    row = torch.stack([r, c], 1).reshape(-1)
    col = torch.stack([c, r], 1).reshape(-1)
    eid = torch.stack([e, e], 1).reshape(-1)
    out = {"nodes": nodes, "row": row, "col": col, "eids": eid, "dist_to_src": None, "dist_to_dst": None}
    if need_dist and n >= 2:
        d_dst = _bfs(n, row, col, start=1, removed=0)
        d_src = _bfs(n, row, col, start=0, removed=1)
        d_dst[0] = 0
        d_src[1] = 0
        out["dist_to_src"], out["dist_to_dst"] = d_src, d_dst
    return out
