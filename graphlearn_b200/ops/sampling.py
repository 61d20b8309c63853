"""Neighbor sampling ops (K1) - dispatch + portable torch implementation.

``sample_neighbors`` picks, per call:
  * the sm_90a peer-memory kernel (csrc/sampling.cu) when the shards live on
    CUDA devices - one launch serves local and remote adjacency rows;
  * otherwise the portable path: hash-partition the seeds, all-to-all them to
    their owners (gloo / NCCL), sample with vectorised torch ops on the local
    shard and stitch the answers back (= the reference's per-hop RPC pattern,
    graphlearn/src/core/runner/op_runner.h:60-152).  This path is also the
    numerics/semantics oracle for the kernels.

Strategy names and semantics follow graphlearn/python/gsl/dag_node.py:197-210
and graphlearn/src/core/operator/sampler/*.cc.
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch

from .. import config as _config
from ..parallel import partition as part
from ..parallel.runtime import native
from ..store.shards import CsrShard
from . import rng as _rng

STRATEGY = {
    "random": 0,
    "random_without_replacement": 1,
    "topk": 2,
    "edge_weight": 3,
    "in_degree": 3,
}
FILTER_NONE, FILTER_ID, FILTER_TS = 0, 1, 2


def _eid_of(csr: CsrShard, pos: torch.Tensor) -> torch.Tensor:
    """edge id of a CSR position: the position itself, or the explicit id column of in-edge CSRs."""
    e = getattr(csr, "eids", None)
    if e is None or e.local.numel() == 0:
        return pos
    return e.local[pos.clamp(max=e.local.numel() - 1)]


def _local_sample(csr: CsrShard, vids: torch.Tensor, k: int, strategy: str, filter_mode: int,
                  fvals: Optional[torch.Tensor], circular: bool, default_id: int,
                  gen: Optional[torch.Generator]) -> Tuple[torch.Tensor, torch.Tensor]:
    """Sample for seeds OWNED by this rank using torch ops only."""
    W = csr.rt.world
    dev = vids.device
    B = int(vids.numel())
    indptr, indices = csr.indptr.local, csr.indices.local
    rows = torch.div(vids, W, rounding_mode="floor")
    ok = (vids >= 0) & (rows < csr.n_src_rows)
    rows_c = torch.where(ok, rows, torch.zeros_like(rows))
    beg = indptr[rows_c]
    deg = torch.where(ok, indptr[rows_c + 1] - beg, torch.zeros_like(beg))
    nbr = torch.full((B, k), default_id, dtype=torch.int64, device=dev)
    eid = torch.full((B, k), -1, dtype=torch.int64, device=dev)
    if B == 0 or k == 0:
        return nbr, eid
    if filter_mode == FILTER_ID:
        # exact reference semantics: drop hits first, then order / pad
        return _local_sample_idfilter(csr, vids, k, strategy, fvals, circular, default_id, gen)
    m = deg.clone()
    reversed_ = False
    if filter_mode == FILTER_TS and csr.ts is not None:
        ts = csr.ts.local
        # per-row count of edges with ts < bound (rows are ts-ascending; strict like the reference's
        # accelerated path, filter.cc:68-82,193-228)
        maxd = int(deg.max().item()) if B > 0 else 0
        ar = torch.arange(max(maxd, 1), device=dev)
        pos = (beg[:, None] + ar[None, :]).clamp_(max=max(ts.numel() - 1, 0))
        inrow = ar[None, :] < deg[:, None]
        m = ((ts[pos] < fvals[:, None]) & inrow).sum(1) if ts.numel() > 0 else torch.zeros_like(deg)
        reversed_ = True
    rnd = lambda *shape: torch.rand(*shape, device=dev, generator=gen)  # noqa: E731
    j = torch.arange(k, device=dev)[None, :].expand(B, k)
    has = m > 0
    mm = m.clamp(min=1)[:, None]
    if strategy == "random":
        pick = torch.minimum((rnd(B, k) * mm).long(), mm - 1)
        valid = has[:, None].expand(B, k).clone()
    elif strategy in ("edge_weight", "in_degree"):
        cum_t = csr.cumw if strategy == "edge_weight" else csr.cumw_indeg
        assert cum_t is not None, "weighted sampling needs per-edge weights"
        cum = cum_t.local
        last = (beg + mm[:, 0] - 1).clamp_(min=0, max=max(cum.numel() - 1, 0))
        total = cum[last] if cum.numel() > 0 else torch.zeros(B, device=dev)
        target = rnd(B, k) * total[:, None]
        maxd = int(m.max().item())
        ar = torch.arange(max(maxd, 1), device=dev)
        pos = (beg[:, None] + ar[None, :]).clamp_(max=max(cum.numel() - 1, 0))
        rowcum = torch.where(ar[None, :] < m[:, None], cum[pos] if cum.numel() > 0 else torch.zeros(B, 1, device=dev),
                             torch.full((1, 1), float("inf"), device=dev))
        pick = (rowcum[:, None, :] <= target[:, :, None]).sum(-1).minimum(mm - 1)
        valid = has[:, None].expand(B, k).clone()
    else:
        # ordered strategies
        if strategy == "random_without_replacement":
            maxd = int(m.max().item())
            keys = rnd(B, max(maxd, 1))
            keys = torch.where(torch.arange(max(maxd, 1), device=dev)[None, :] < m[:, None], keys,
                               torch.full_like(keys, 2.0))
            perm = torch.argsort(keys, dim=1)            # random order of the valid prefix
            jj = torch.where(j < mm, j, j % mm) if circular else j
            pick = torch.gather(perm, 1, jj.clamp(max=max(maxd, 1) - 1))
        else:  # topk
            pick = torch.where(j < mm, j, j % mm) if circular else j.clone()
        valid = has[:, None] & ((j < m[:, None]) | circular)
        if reversed_:
            pick = (mm - 1 - pick).clamp_(min=0)
    pos = (beg[:, None] + pick).clamp_(min=0, max=max(indices.numel() - 1, 0))
    if indices.numel() > 0:
        nbr = torch.where(valid, indices[pos], nbr)
        eid = torch.where(valid, _eid_of(csr, pos), eid)
    return nbr, eid


def _local_sample_idfilter(csr, vids, k, strategy, fvals, circular, default_id, gen):
    """Row-by-row reference implementation for the (rare) id-filtered case."""
    W = csr.rt.world
    indptr, indices = csr.indptr.local.cpu(), csr.indices.local.cpu()
    cum = None
    if strategy in ("edge_weight", "in_degree"):
        cum = (csr.cumw if strategy == "edge_weight" else csr.cumw_indeg).local.cpu()
    B = int(vids.numel())
    nbr = torch.full((B, k), default_id, dtype=torch.int64)
    eid = torch.full((B, k), -1, dtype=torch.int64)
    g = torch.Generator()
    g.manual_seed(int(torch.randint(0, 2 ** 31 - 1, (1,), generator=gen, device=vids.device).item()) if gen is not None else 0)
    vc, fc = vids.cpu(), fvals.cpu()
    for b in range(B):
        v = int(vc[b])
        row = v // W
        if v < 0 or row >= csr.n_src_rows:
            continue
        s, e = int(indptr[row]), int(indptr[row + 1])
        cand = [i for i in range(s, e) if int(indices[i]) != int(fc[b])]
        if not cand:
            continue
        if strategy == "random":
            sel = [cand[int(torch.randint(0, len(cand), (1,), generator=g))] for _ in range(k)]
        elif strategy in ("edge_weight", "in_degree"):
            w = torch.tensor([float(cum[i] - (cum[i - 1] if i > s else 0.0)) for i in cand])
            sel = [cand[int(i)] for i in torch.multinomial(w.clamp(min=1e-12), k, replacement=True, generator=g)]
        else:
            if strategy == "random_without_replacement":
                cand = [cand[int(i)] for i in torch.randperm(len(cand), generator=g)]
            sel = [cand[i % len(cand)] if (i < len(cand) or circular) else -1 for i in range(k)]
        for jx, i in enumerate(sel):
            if i >= 0:
                nbr[b, jx] = indices[i]
                eid[b, jx] = i
    eid = eid.to(vids.device)
    eid = torch.where(eid >= 0, _eid_of(csr, eid.clamp(min=0)), eid)
    return nbr.to(vids.device), eid


# ---------------------------------------------------------------------- user-defined samplers
# The reference lets users add operators in C++: subclass Operator / Sampler, implement the LOCAL ``Process`` and
# ``REGISTER_OPERATOR("xxxSampler", ...)``; the framework partitions the request over the servers and stitches the answers
# (docs/en/gl/developer/operator.md, src/core/operator/operator.h, op_registry).  The same contract here: register the local
# rule, ``g.V(..).outV(e).sample(k).by("xxx")`` / ``g.neighbor_sampler(e, k, strategy="xxx")`` run it on the owner of every
# source row (Partition -> all-to-all -> local rule -> Stitch on multi-rank jobs).
_CUSTOM_SAMPLERS = {}


class LocalAdjacency(object):
    """What a custom sampling rule sees: this rank's CSR shard.  Row r holds positions ``indptr[r] .. indptr[r + 1] - 1`` of
    ``indices`` (destination ids in the engine's virtual-id space), ``weights`` / ``timestamps`` (or None); rows are ordered by
    weight descending, or by timestamp ascending for timestamped edge types."""

    def __init__(self, csr: CsrShard):
        self.edge_type, self.num_rows, self.num_edges = csr.type, csr.n_src_rows, csr.n_edges
        self.indptr, self.indices = csr.indptr.local, csr.indices.local
        self.weights = csr.weights.local if csr.weights is not None else None
        self.timestamps = csr.ts.local if csr.ts is not None else None

    def degrees(self, rows: torch.Tensor) -> torch.Tensor:
        return self.indptr[rows + 1] - self.indptr[rows]


def register_sampler(name: str, fn, overwrite: bool = False):
    """Register a neighbour-sampling strategy ``name``.

    ``fn(adj: LocalAdjacency, rows: int64 [n], k: int, generator: torch.Generator | None) -> int64 [n, k]`` returns, for every
    local source row, k POSITIONS into ``adj.indices`` taken from that row's range (``-1`` = no neighbour: the slot gets the
    default neighbour id).  Positions outside the row are treated as -1, so a rule can never fabricate an edge."""
    if not callable(fn):
        raise ValueError("fn must be callable")
    if name in STRATEGY or name == "full":
        raise ValueError("%r is a built-in strategy" % (name,))
    if name in _CUSTOM_SAMPLERS and not overwrite:
        raise ValueError("sampler %r is already registered" % (name,))
    _CUSTOM_SAMPLERS[name] = fn
    return fn


def unregister_sampler(name: str):
    _CUSTOM_SAMPLERS.pop(name, None)


def registered_samplers():
    return sorted(_CUSTOM_SAMPLERS)


def _custom_sample(csr: CsrShard, src: torch.Tensor, k: int, strategy: str, gen, default_id: int):
    fn = _CUSTOM_SAMPLERS[strategy]
    W = csr.rt.world
    adj = LocalAdjacency(csr)

    def run(v):
        rows = torch.div(v, W, rounding_mode="floor")
        ok = (v >= 0) & (rows < csr.n_src_rows)
        rows = torch.where(ok, rows, torch.zeros_like(rows))
        n = int(v.numel())
        if n == 0 or csr.n_src_rows == 0:
            return (torch.full((n, k), default_id, dtype=torch.int64, device=v.device),
                    torch.full((n, k), -1, dtype=torch.int64, device=v.device))
        pos = torch.as_tensor(fn(adj, rows, int(k), gen)).to(torch.int64).to(v.device)
        if tuple(pos.shape) != (n, k):
            raise ValueError("sampler %r returned shape %s, expected %s" % (strategy, tuple(pos.shape), (n, k)))
        beg, end = adj.indptr[rows], adj.indptr[rows + 1]
        valid = ok[:, None] & (pos >= beg[:, None]) & (pos < end[:, None])
        p = pos.clamp(min=0, max=max(csr.n_edges - 1, 0))
        if csr.n_edges == 0:
            valid = torch.zeros_like(valid)
            nbr_raw = torch.zeros_like(p)
            eid_raw = torch.zeros_like(p)
        else:
            nbr_raw, eid_raw = adj.indices[p], _eid_of(csr, p)
        return (torch.where(valid, nbr_raw, torch.full_like(p, default_id)), torch.where(valid, eid_raw, torch.full_like(p, -1)))
    return part.remote_apply(src, run, W, ())


def sample_neighbors(csr: CsrShard, src_vids: torch.Tensor, k: int, strategy: str = "random",
                     filter_mode: int = FILTER_NONE, filter_values: Optional[torch.Tensor] = None,
                     want_eids: bool = True, rng: Optional["_rng.DeviceRng"] = None, salt: int = 0,
                     padding_circular: Optional[bool] = None, out: Optional[torch.Tensor] = None):
    """src_vids: int64 [B] -> (nbr_vids [B, k], edge_ids [B, k] | None).  ``out`` (CUDA kernel path): a
    pre-allocated contiguous int64 buffer of B*k elements the neighbour ids are written into (static-shape
    engines sample straight into their hop buffers - no copy kernel)."""
    cfg = _config.get()
    circular = (cfg.padding_mode == _config.PADDING_CIRCULAR) if padding_circular is None else padding_circular
    if strategy == "full":
        raise ValueError("use sample_full for the 'full' strategy")
    src = src_vids.reshape(-1).to(torch.int64)
    rng = rng or _rng.default_rng(csr.rt)
    if strategy in _CUSTOM_SAMPLERS:
        if filter_mode != FILTER_NONE:
            raise ValueError("filters are not available for user-defined samplers (filter inside the rule)")
        nbr, eid = _custom_sample(csr, src, int(k), strategy, rng.torch_generator(salt), int(cfg.default_neighbor_id))
        if out is not None:
            out.view(-1).copy_(nbr.reshape(-1))
        return nbr, (eid if want_eids else None)
    if strategy == "edge_weight" and csr.cumw is None:
        strategy = "random"        # unweighted edge type: every edge carries the same default weight (the reference's behaviour)
    if strategy not in STRATEGY:
        raise ValueError("unknown sampling strategy %r (built-in: %s; registered: %s)" % (strategy, ", ".join(STRATEGY),
                                                                                          ", ".join(registered_samplers()) or "-"))
    if csr.rt.is_cuda and cfg.use_peer_kernels:
        desc = csr.desc_indeg if strategy == "in_degree" else csr.desc
        if strategy == "in_degree" and desc is None:
            raise ValueError("in_degree sampling needs in-degree weights (CsrShard.set_indegree_weights)")
        nbr, eid = native().sample_neighbors(desc, src, int(k), STRATEGY[strategy], int(filter_mode), filter_values,
                                             bool(circular), int(cfg.sampling_retry_times),
                                             int(cfg.default_neighbor_id), rng.state, int(salt), bool(want_eids), out)
        return nbr, (eid if want_eids else None)
    gen = rng.torch_generator(salt)
    extra = (filter_values.reshape(-1),) if filter_mode != FILTER_NONE else ()

    def fn(v, *ex):
        return _local_sample(csr, v, k, strategy, filter_mode, ex[0] if ex else None, circular,
                             cfg.default_neighbor_id, gen)

    nbr, eid = part.remote_apply(src, fn, csr.rt.world, extra)
    if out is not None:
        out.view(-1).copy_(nbr.reshape(-1))
    return nbr, (eid if want_eids else None)


def get_degrees(csr: CsrShard, src_vids: torch.Tensor, cap: int = 0) -> torch.Tensor:
    src = src_vids.reshape(-1).to(torch.int64)
    if csr.rt.is_cuda and _config.get().use_peer_kernels:
        return native().get_degrees(csr.desc, src, int(cap))
    W = csr.rt.world

    def fn(v):
        rows = torch.div(v, W, rounding_mode="floor")
        ok = (v >= 0) & (rows < csr.n_src_rows)
        rc = torch.where(ok, rows, torch.zeros_like(rows))
        ip = csr.indptr.local
        d = torch.where(ok, ip[rc + 1] - ip[rc], torch.zeros_like(rc))
        if cap > 0:
            d = d.clamp(max=cap)
        return (d,)

    return part.remote_apply(src, fn, W)[0]


def sample_full(csr: CsrShard, src_vids: torch.Tensor, cap: int = 0, want_eids: bool = True, max_total: int = 0):
    """FullSampler: sparse output (values, eids, offsets[B+1])
    (graphlearn/src/core/operator/sampler/full_sampler.cc:43-88).  ``max_total`` > 0 (CUDA): sync-free mode - outputs
    have that fixed capacity (-1 padded, rows truncated when the data needs more), nothing is read back on the host,
    so the op is CUDA-graph capturable; ``offsets[B]`` holds the produced count on the device."""
    src = src_vids.reshape(-1).to(torch.int64)
    if csr.rt.is_cuda and _config.get().use_peer_kernels:
        vals, eids, offsets = native().sample_full(csr.desc, src, int(cap), bool(want_eids), int(max_total))
        return vals, (eids if want_eids else None), offsets
    W = csr.rt.world
    deg = get_degrees(csr, src, cap)
    B = int(src.numel())
    offsets = torch.zeros(B + 1, dtype=torch.int64, device=src.device)
    offsets[1:] = torch.cumsum(deg, 0)
    maxd_t = deg.max().reshape(1) if B > 0 else torch.zeros(1, dtype=torch.int64, device=src.device)
    if W > 1:       # every owner must answer with the same row width
        import torch.distributed as dist
        dist.all_reduce(maxd_t, op=dist.ReduceOp.MAX)
    maxd = int(maxd_t.item())
    if maxd == 0:
        z = torch.zeros(0, dtype=torch.int64, device=src.device)
        return z, (z.clone() if want_eids else None), offsets

    def fn(v):
        rows = torch.div(v, W, rounding_mode="floor")
        ok = (v >= 0) & (rows < csr.n_src_rows)
        rc = torch.where(ok, rows, torch.zeros_like(rows))
        ip, idx = csr.indptr.local, csr.indices.local
        beg = ip[rc]
        ar = torch.arange(maxd, device=v.device)
        pos = (beg[:, None] + ar[None, :]).clamp_(max=max(idx.numel() - 1, 0))
        return (idx[pos] if idx.numel() > 0 else torch.zeros(v.numel(), maxd, dtype=torch.int64, device=v.device),
                _eid_of(csr, pos))

    dense_n, dense_e = part.remote_apply(src, fn, W)
    mask = torch.arange(maxd, device=src.device)[None, :] < deg[:, None]
    return dense_n[mask], (dense_e[mask] if want_eids else None), offsets
