"""Negative samplers (K2).

Semantics follow the reference operators:
  random      uniform over the destination candidates, NOT guaranteed negative
              (graphlearn/src/core/operator/sampler/random_negative_sampler.cc:46-58)
  in_degree   dst drawn ~ in-degree, true neighbours of src rejected, strictness
              dropped after `neg_sampling_retry_times` rounds
              (in_degree_negative_sampler.cc:61-98)
  node_weight node drawn ~ node weight, ids of the src batch rejected
              (node_weight_negative_sampler.cc:61-92)
  conditional negatives sharing selected attribute values with the positive dst
              (conditional_negative_sampler.cc:37-156)

GPU design: instead of Vose alias tables (alias_method.cc:57-123) the weighted
draws use one global inclusive prefix-sum per (shard, distribution) and a
binary search (``torch.searchsorted`` -> a single vectorised device kernel);
rejection is a sorted-row membership test against the CSR (rows are fetched
with the peer-memory full sampler when the source is remote).  The candidate
universe is the WHOLE destination node type, not only the local shard's dst
list as in the reference (its quirk listed in SURVEY Appendix B).
"""
from __future__ import annotations

from typing import Dict, Optional

import torch

from .. import config as _config
from . import gather as G
from . import sampling as S


def _draw_global_uniform(tab, B, k, gen, device):
    """uniform vids over all rows of all ranks of a node table."""
    W = tab.rt.world
    nrows = torch.tensor(tab.nrows, device=device, dtype=torch.int64)
    cum = torch.cumsum(nrows, 0)
    total = int(cum[-1].item())
    if total == 0:
        return torch.full((B, k), -1, dtype=torch.int64, device=device)
    u = torch.randint(0, total, (B, k), device=device, generator=gen)
    owner = torch.searchsorted(cum, u, right=True)
    row = u - (cum[owner] - nrows[owner])
    return row * W + owner


class _WeightedSampler(object):
    """draw vids ~ weight over a sharded node table (weights gathered once to every rank: they are
    [N] floats - small next to the feature table)."""

    def __init__(self, rt, weights_local: torch.Tensor):
        W = rt.world
        if W > 1:
            import torch.distributed as dist
            sizes = rt.all_gather_object(int(weights_local.numel()))
            mx = max(sizes)
            pad = torch.zeros(mx, device=weights_local.device, dtype=torch.float32)
            pad[:weights_local.numel()] = weights_local.float()
            allw = [torch.zeros_like(pad) for _ in range(W)]
            dist.all_gather(allw, pad)
            parts = [a[:n] for a, n in zip(allw, sizes)]
        else:
            sizes = [int(weights_local.numel())]
            parts = [weights_local.float()]
        self.sizes = sizes
        self.W = W
        w = torch.cat(parts).clamp(min=0).double()
        self.cum = torch.cumsum(w, 0)
        self.total = float(self.cum[-1].item()) if w.numel() else 0.0
        self.offsets = torch.tensor([0] + list(torch.tensor(sizes).cumsum(0).tolist()), device=w.device)

    def draw(self, shape, gen, device):
        if self.total <= 0:
            return torch.full(shape, -1, dtype=torch.int64, device=device)
        u = torch.rand(shape, device=device, generator=gen, dtype=torch.float64) * self.total
        pos = torch.searchsorted(self.cum, u, right=True).clamp_(max=self.cum.numel() - 1)
        owner = torch.searchsorted(self.offsets[1:], pos, right=True)
        row = pos - self.offsets[owner]
        return row * self.W + owner


def _cache_of(store) -> Dict[tuple, "_WeightedSampler"]:
    """Weighted-sampler cache of ONE graph store (reference: AliasMethodFactory caches per edge type inside a server
    process, in_degree_negative_sampler.cc:61-98).  It lives on the store object so that a second Graph with the same
    type names - or a rebuilt one - can never see a stale distribution."""
    c = getattr(store, "_neg_cache", None)
    if c is None:
        c = {}
        store._neg_cache = c
    return c


def _is_neighbor(csr, src_v: torch.Tensor, cand: torch.Tensor) -> torch.Tensor:
    """[B, k] bool: cand[b, j] in adj(src[b]).  Rows come from the (peer capable) full sampler."""
    vals, _, offs = S.sample_full(csr, src_v, cap=0, want_eids=False)
    B, k = cand.shape
    counts = offs[1:] - offs[:-1]
    if vals.numel() == 0:
        return torch.zeros_like(cand, dtype=torch.bool)
    seg = torch.repeat_interleave(torch.arange(B, device=cand.device), counts)
    # hash (segment, value) pairs into sortable keys
    base = int(max(int(vals.max().item()), int(cand.max().item())) + 2)
    keys = torch.sort(seg * base + (vals + 1))[0]
    q = torch.arange(B, device=cand.device)[:, None] * base + (cand + 1)
    pos = torch.searchsorted(keys, q.reshape(-1)).clamp_(max=keys.numel() - 1)
    return (keys[pos] == q.reshape(-1)).reshape(B, k)


def _shard_offsets(tab, device):
    off = [0]
    for n in tab.nrows:
        off.append(off[-1] + int(n))
    return torch.tensor(off, dtype=torch.int64, device=device), off[-1]


def edge_negative(store, etype: str, src_v: torch.Tensor, k: int, strategy: str, gen, direction: str = "out",
                  rng=None, salt: int = 0):
    cfg = _config.get()
    csr = store.edges[etype] if direction == "out" else store.reverse_csr(etype)
    dst_tab = store.nodes[csr.dst_type]
    B = int(src_v.numel())
    dev = src_v.device
    if store.rt.is_cuda and cfg.use_peer_kernels and rng is not None and strategy in ("random", "in_degree"):
        # K2 kernel: candidate draw + neighbour rejection against the (peer-mapped) CSR in one launch
        from ..parallel.runtime import native
        cum = None
        if strategy == "in_degree":
            key = ("indeg", etype, direction)
            if key not in _cache_of(store):
                if direction == "out":
                    store.reverse_csr(etype)
                    wloc = dst_tab.in_degrees[etype].float()
                else:
                    wloc = store.nodes[csr.dst_type].out_degrees[etype].float()
                _cache_of(store)[key] = _WeightedSampler(store.rt, wloc)
            cum = _cache_of(store)[key].cum
        off, total = _shard_offsets(dst_tab, dev)
        if total == 0:
            return torch.full((B, k), -1, dtype=torch.int64, device=dev)
        return native().negative_sample(csr.desc, src_v.reshape(-1), int(k), cum, off, int(total),
                                        strategy == "in_degree", int(cfg.neg_sampling_retry_times), 1024,
                                        rng.state, int(salt), None)
    if strategy == "random":
        return _draw_global_uniform(dst_tab, B, k, gen, dev)
    if strategy == "in_degree":
        key = ("indeg", etype, direction)
        if key not in _cache_of(store):
            if direction == "out":
                store.reverse_csr(etype)
                wloc = dst_tab.in_degrees[etype].float()
            else:
                wloc = store.nodes[csr.dst_type].out_degrees[etype].float()
            _cache_of(store)[key] = _WeightedSampler(store.rt, wloc)
        ws = _cache_of(store)[key]
        neg = ws.draw((B, k), gen, dev)
        for _ in range(max(1, cfg.neg_sampling_retry_times)):
            bad = _is_neighbor(csr, src_v, neg)             # collective when world > 1
            any_bad = bad.any().to(torch.int32).reshape(1)
            if store.rt.world > 1:                          # every rank must run the same number of rounds
                import torch.distributed as dist
                dist.all_reduce(any_bad, op=dist.ReduceOp.MAX)
            if int(any_bad.item()) == 0:
                break
            redraw = ws.draw((B, k), gen, dev)
            neg = torch.where(bad, redraw, neg)
        return neg
    raise ValueError("unknown negative sampling strategy %r" % (strategy,))


def node_weight_negative(store, ntype: str, src_v: torch.Tensor, k: int, gen):
    cfg = _config.get()
    tab = store.nodes[ntype]
    B = int(src_v.numel())
    dev = src_v.device
    if tab.weights is None:
        return _draw_global_uniform(tab, B, k, gen, dev)
    key = ("nw", ntype)
    if key not in _cache_of(store):
        _cache_of(store)[key] = _WeightedSampler(store.rt, tab.weights.local)
    ws = _cache_of(store)[key]
    neg = ws.draw((B, k), gen, dev)
    batch = torch.sort(torch.unique(src_v))[0]
    for _ in range(max(1, cfg.neg_sampling_retry_times)):
        pos = torch.searchsorted(batch, neg.reshape(-1)).clamp_(max=max(batch.numel() - 1, 0))
        bad = (batch[pos] == neg.reshape(-1)).reshape(B, k) if batch.numel() else torch.zeros_like(neg, dtype=torch.bool)
        if not bool(bad.any()):
            break
        neg = torch.where(bad, ws.draw((B, k), gen, dev), neg)
    return neg


def conditional_negative(store, etype: str, src_v: torch.Tensor, dst_v: torch.Tensor, k: int, strategy: str,
                         cond: dict, gen):
    """Negatives that share selected int / float attribute columns with the positive dst; each
    selected column gets ``prop`` of the k slots, the remainder is filled by the base strategy
    (conditional_negative_sampler.cc:37-156).  True neighbours of src and (unique=True)
    duplicates are avoided on a best-effort basis like the reference."""
    cfg = _config.get()
    is_edge = etype in store.edges
    if not is_edge and etype not in store.nodes:
        raise KeyError("conditional negative sampling: %r is neither an edge type nor a node type" % (etype,))
    csr = store.edges[etype] if is_edge else None
    dst_type = csr.dst_type if is_edge else etype
    tab = store.nodes[dst_type]
    rt = store.rt
    B = int(src_v.numel())
    dev = src_v.device
    base_strategy = strategy if strategy in ("random", "in_degree") else "random"
    if is_edge:
        def _base():
            return edge_negative(store, etype, src_v, k, base_strategy, gen)
    else:
        # object = a NODE type (``negative_sampler(node_type, strategy="node_weight", conditional=True)``): candidates are the
        # nodes of that type drawn by weight (uniformly when the table has no weights); there is no neighbourhood to avoid,
        # only the positive ids
        def _base():
            return node_weight_negative(store, etype, dst_v, k, gen)
    out = _base()
    cols = [("int", c, p) for c, p in zip(cond.get("int_cols", []), cond.get("int_props", []))] + \
           [("float", c, p) for c, p in zip(cond.get("float_cols", []), cond.get("float_props", []))] + \
           [("str", c, p) for c, p in zip(cond.get("str_cols", []), cond.get("str_props", []))]
    batch_share = bool(cond.get("batch_share"))
    if batch_share:
        # the exclusion set is the batch's positive dst ids, shared by every row, instead of each
        # row's own neighbourhood (conditional_negative_sampler.cc:113-126)
        pos_sorted = torch.sort(torch.unique(dst_v))[0]

        def _excluded(cand):
            pos = torch.searchsorted(pos_sorted, cand.reshape(-1)).clamp_(max=max(pos_sorted.numel() - 1, 0))
            return (pos_sorted[pos] == cand.reshape(-1)).reshape(cand.shape)
        for _ in range(max(1, int(cfg.neg_sampling_retry_times))):       # strictness is dropped after the retries
            out = torch.where(_excluded(out), _base(), out)
    elif is_edge:
        def _excluded(cand):
            return _is_neighbor(csr, src_v, cand) | (cand == dst_v[:, None])
    else:
        def _excluded(cand):
            return cand == dst_v[:, None]
    if not cols:
        return out
    slot = 0
    for kind, c, prop in cols:
        n_slots = int(round(prop * k))
        if n_slots <= 0 or slot >= k:
            continue
        n_slots = min(n_slots, k - slot)
        if kind == "str":
            # string attributes live on the host of the owning rank: factorise the local column and the
            # positives' values into integer codes, then reuse the sorted-run index below
            import numpy as np
            if tab.str_dim == 0:
                raise ValueError("conditional negative sampling: node type %r has no string attributes" % (dst_type,))
            # factorise the LOCAL column and the positives' values (fetched from their owners) with one shared
            # vocabulary, then reuse the sorted-run index below
            col = np.asarray(tab.strings[:, c], dtype=object).astype(str) if tab.strings is not None and tab.n_local else \
                np.zeros(0, dtype=str)
            want = tab.lookup_strings(dst_v, cfg.default_string_attribute)[:, c].astype(str)
            vocab, codes = np.unique(np.concatenate([col, want]), return_inverse=True)
            local_vals = torch.as_tensor(codes[:len(col)], device=dev).long()
            dstv = torch.as_tensor(codes[len(col):], device=dev).long()
        elif kind == "int":
            if tab.ints is None:
                raise ValueError("conditional negative sampling: node type %r has no int attributes" % (dst_type,))
            attr_all = tab.ints
            dstv = G.gather_any(rt, attr_all, dst_v, fill=0)[:, c]
            local_vals = attr_all.local[:, c]
        else:
            if tab.feats is None:
                raise ValueError("conditional negative sampling: node type %r has no float attributes" % (dst_type,))
            dstv = G.gather_rows(rt, tab.feats, tab.feat_desc, dst_v, tab.float_dim)[:, c]
            local_vals = tab.feats.local[:, c].float()
        # inverted index over the LOCAL shard: sort rows by attribute value, pick uniformly inside
        # the run of equal values (the reference's AttributeNodesMap)
        order = torch.argsort(local_vals, stable=True)
        sv = local_vals[order]
        key = dstv.to(sv.dtype).contiguous()
        lo = torch.searchsorted(sv, key, right=False)
        hi = torch.searchsorted(sv, key, right=True)
        span = (hi - lo)
        ok = (span > 0)[:, None].expand(B, n_slots)
        chosen = out[:, slot:slot + n_slots].clone()
        todo = ok.clone()
        # redraw excluded candidates for a few rounds before leaving a slot to the base strategy
        # (the reference's ConditionTable::Sample skips ids of the exclusion set while filling the quota)
        for _ in range(max(1, int(cfg.neg_sampling_retry_times)) + 1):
            u = torch.rand(B, n_slots, device=dev, generator=gen)
            pick = lo[:, None] + (u * span[:, None].clamp(min=1).float()).long()
            pick = torch.minimum(pick, (hi - 1).clamp(min=0)[:, None]).clamp_(min=0, max=max(order.numel() - 1, 0))
            cand = order[pick] * rt.world + rt.rank if order.numel() else torch.full((B, n_slots), -1, device=dev)
            good = todo & ~_excluded(cand)       # `_excluded` is collective on > 1 rank: fixed round count
            if cond.get("unique"):
                # a candidate already chosen in another slot of the row is not "good" either
                dupe = (cand.unsqueeze(2) == chosen.unsqueeze(1)).any(2)
                good &= ~dupe
                # and keep only the first of equal candidates inside this round
                srt, idx = torch.sort(torch.where(good, cand, torch.full_like(cand, -1)), dim=1, stable=True)
                rep = torch.zeros_like(good)
                rep[:, 1:] = (srt[:, 1:] == srt[:, :-1]) & (srt[:, 1:] >= 0)
                good &= ~torch.zeros_like(good).scatter(1, idx, rep)
            chosen = torch.where(good, cand, chosen)
            todo &= ~good
        out[:, slot:slot + n_slots] = chosen
        slot += n_slots
    if cond.get("unique"):
        # replace in-row duplicates by fresh base draws (best effort, one round)
        srt, idx = torch.sort(out, dim=1)
        dup = torch.zeros_like(out, dtype=torch.bool)
        dup[:, 1:] = srt[:, 1:] == srt[:, :-1]
        dup = torch.zeros_like(out, dtype=torch.bool).scatter(1, idx, dup)
        fresh = _base()
        out = torch.where(dup, fresh, out)
    return out
