"""K10: KNN over a node type's float attributes - flat and IVF-flat indexes.

The reference wraps faiss indexes (flat / ivfflat / ivfpq, CPU or GPU) behind ``KnnOperator``: the query is
broadcast to every server and the per-server top-k lists are merged with a k-heap
(graphlearn/src/contrib/knn/index_factory.cc:28-50, knn_request.cc:96-111,167-202).  Here:

* **flat** - ``csrc/knn.cu``: one kernel per 128-query tile streams the shard through a wgmma score GEMM with a
  fused running top-k (the [B, N] score matrix never exists), a second kernel merges the per-SM lists; the
  candidates (2k, scored from bf16 operands) are re-ranked in fp32 so the result equals an fp32 brute force;
* **ivfflat** - k-means coarse quantiser at build time, inverted lists = a row permutation; a query probes its
  ``nprobe`` nearest lists with the same kernel (row-index-list mode);
* **ivfpq** - the same coarse quantiser, rows stored as ``m`` one-byte product-quantiser codes of their residual to
  the list centroid; ``knn_ivfpq_scan_kernel`` builds the asymmetric-distance table of a (query, list) pair in shared
  memory and scores a row with ``m`` look-ups; the best candidates are re-ranked with the exact rows (they stay in
  HBM anyway), so reported distances are exact;
* multi-GPU: every rank searches its shard, writes its list into a symmetric buffer and merges all peers' lists
  with peer loads over NVLink (no NCCL on the data path).

Metric 0 = L2 (distances are squared), 1 = inner product (``gl.set_knn_metric``).  The portable torch path below
is the CPU implementation and the numerics oracle.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from .. import config as _config


class KnnOption(object):
    def __init__(self, k=1):
        self.k = int(k)


def _shard_topk(x: torch.Tensor, q: torch.Tensor, k: int, metric: int, chunk: int = 1 << 18):
    """portable path: chunked GEMM + topk"""
    n = x.size(0)
    best_s = torch.full((q.size(0), k), float("-inf"), device=q.device)
    best_i = torch.full((q.size(0), k), -1, dtype=torch.int64, device=q.device)
    qn = (q * q).sum(1, keepdim=True)
    for s in range(0, n, chunk):
        xs = x[s:s + chunk].to(q.dtype)
        ip = q @ xs.t()
        score = ip if metric == 1 else -(qn - 2 * ip + (xs * xs).sum(1)[None, :])
        kk = min(k, score.size(1))
        v, i = torch.topk(score, kk, dim=1)
        cat_s = torch.cat([best_s, v], 1)
        cat_i = torch.cat([best_i, i + s], 1)
        v2, j = torch.topk(cat_s, k, dim=1)
        best_s, best_i = v2, torch.gather(cat_i, 1, j)
    return best_s, best_i


def _use_kernel(rt, x) -> bool:
    return rt.is_cuda and _config.get().use_peer_kernels and x.size(1) <= 512


def _norms(table, x):
    """|x|^2 per local row, cached on the table (rebuilt when the table object changes)."""
    c = getattr(table, "_knn_norm", None)
    if c is None or c.numel() != x.size(0):
        c = (x.float() ** 2).sum(1).contiguous()
        table._knn_norm = c
    return c


def _kernel_topk(table, x_full: torch.Tensor, dim: int, q: torch.Tensor, k: int, metric: int, row_list: Optional[torch.Tensor] = None):
    """(score [B, k], rows [B, k]) exact in fp32: the fused kernel proposes kk = min(64, 2k + 8) candidates per query from
    bf16 operands, their true fp32 scores are recomputed on the few gathered rows and the best k kept."""
    from ..parallel.runtime import native
    C = native()
    B = q.size(0)
    dpad = (dim + 63) // 64 * 64
    kk = min(64, max(2 * k + 8, k))
    n_avail = x_full.size(0) if row_list is None else int(row_list.numel())
    kk = max(min(kk, max(n_avail, 1)), min(k, 64))
    norms = _norms(table, x_full[:, :dim]) if metric == 0 else None
    out_s, out_i = [], []
    for s in range(0, B, 128):
        qt = q[s:s + 128]
        bt = qt.size(0)
        qp = torch.zeros(128, dpad, dtype=torch.bfloat16, device=q.device)
        qp[:bt, :dim] = qt
        _, rows = C.knn_flat_topk(x_full, dim, norms, row_list, qp, bt, kk)
        ok = rows >= 0
        xr = x_full[rows.clamp(min=0), :dim].float()                     # [bt, kk, d]
        ip = torch.einsum("bd,bkd->bk", qt.float(), xr)
        sc = ip if metric == 1 else -((qt.float() ** 2).sum(1, keepdim=True) - 2 * ip + (xr ** 2).sum(2))
        sc = torch.where(ok, sc, torch.full_like(sc, float("-inf")))
        v, j = torch.topk(sc, min(k, kk), dim=1)
        r = torch.gather(rows, 1, j)
        if v.size(1) < k:
            pad = k - v.size(1)
            v = torch.cat([v, torch.full((bt, pad), float("-inf"), device=v.device)], 1)
            r = torch.cat([r, torch.full((bt, pad), -1, dtype=torch.int64, device=r.device)], 1)
        out_s.append(v); out_i.append(torch.where(torch.isinf(v), torch.full_like(r, -1), r))
    return torch.cat(out_s), torch.cat(out_i)


class IvfFlatIndex(object):
    """IVF-flat (index_factory.cc:34-38 'ivfflat'): k-means coarse quantiser + inverted lists over ONE shard."""

    def __init__(self, table, x: torch.Tensor, dim: int, nlist: int, nprobe: int, metric: int, iters: int = 8, seed: int = 0):
        self.table, self.x, self.dim, self.metric = table, x, dim, metric
        n = x.size(0)
        self.nlist = max(1, min(int(nlist), max(n, 1)))
        self.nprobe = max(1, min(int(nprobe) if nprobe else max(1, self.nlist // 16), self.nlist))
        g = torch.Generator(device=x.device).manual_seed(seed)
        xf = x[:, :dim].float()
        sample = xf[torch.randperm(n, device=x.device, generator=g)[:min(n, 256 * self.nlist)]] if n > 0 else xf
        cent = sample[torch.randperm(sample.size(0), device=x.device, generator=g)[:self.nlist]].clone() if n > 0 else xf
        for _ in range(iters if n > 0 else 0):
            a = torch.cdist(sample, cent).argmin(1)
            sums = torch.zeros_like(cent).index_add_(0, a, sample)
            cnt = torch.bincount(a, minlength=self.nlist).clamp(min=1).unsqueeze(1)
            cent = torch.where((torch.bincount(a, minlength=self.nlist) > 0).unsqueeze(1), sums / cnt, cent)
        self.centroids = cent.contiguous()
        assign = torch.cat([torch.cdist(xf[s:s + (1 << 18)], cent).argmin(1) for s in range(0, n, 1 << 18)]) if n > 0 else \
            torch.zeros(0, dtype=torch.int64, device=x.device)
        self.order = torch.argsort(assign, stable=True)                  # rows grouped by list
        self.offsets = torch.cat([torch.zeros(1, dtype=torch.int64, device=x.device),
                                  torch.bincount(assign, minlength=self.nlist).cumsum(0)])

    def search(self, q: torch.Tensor, k: int, use_kernel: bool):
        B = q.size(0)
        # nearest lists per query (always by L2 to the centroids, like faiss' IndexIVFFlat quantiser)
        d = torch.cdist(q.float(), self.centroids)
        probes = d.topk(self.nprobe, dim=1, largest=False).indices      # [B, nprobe]
        if use_kernel and self.x.dtype in (torch.float32, torch.bfloat16):
            # one launch: a CTA per (query, probed list) scans the list exactly in fp32, then the shared-memory merge
            from ..parallel.runtime import native
            s, r = native().knn_ivf_search(self.x, self.dim, self.order, self.offsets, q.float().contiguous(), probes.contiguous(),
                                           int(k), int(self.metric))
            s = torch.where(r >= 0, s, torch.full_like(s, float("-inf")))
            return s, r
        best_s = torch.full((B, k), float("-inf"), device=q.device)
        best_i = torch.full((B, k), -1, dtype=torch.int64, device=q.device)
        offs = self.offsets.tolist()
        for l in torch.unique(probes).tolist():
            qs = (probes == l).any(1).nonzero().flatten()
            lo, hi = offs[l], offs[l + 1]
            if hi == lo or qs.numel() == 0:
                continue
            rows = self.order[lo:hi]
            if use_kernel:
                s, r = _kernel_topk(self.table, self.x, self.dim, q[qs], k, self.metric, row_list=rows)
            else:
                s, r = _shard_topk(self.x[rows, :self.dim].float(), q[qs].float(), min(k, hi - lo), self.metric)
                r = torch.where(r >= 0, rows[r.clamp(min=0)], r)
                if s.size(1) < k:
                    pad = k - s.size(1)
                    s = torch.cat([s, torch.full((s.size(0), pad), float("-inf"), device=s.device)], 1)
                    r = torch.cat([r, torch.full((r.size(0), pad), -1, dtype=torch.int64, device=r.device)], 1)
            cs = torch.cat([best_s[qs], s], 1)
            ci = torch.cat([best_i[qs], r], 1)
            v, j = torch.topk(cs, k, dim=1)
            best_s[qs], best_i[qs] = v, torch.gather(ci, 1, j)
        return best_s, best_i


def _kmeans(x: torch.Tensor, k: int, iters: int, g: torch.Generator) -> torch.Tensor:
    """plain Lloyd iterations on the rows of x -> [k, d] centroids (empty clusters keep their previous centre)."""
    n = x.size(0)
    if n == 0:
        return torch.zeros(k, x.size(1), device=x.device)
    pick = torch.randperm(n, device=x.device, generator=g)[:k]
    cent = x[pick].clone()
    if cent.size(0) < k:                                                 # fewer points than centres: repeat points
        cent = torch.cat([cent, x[torch.randint(0, n, (k - cent.size(0),), device=x.device, generator=g)]])
    for _ in range(iters):
        a = torch.cdist(x, cent).argmin(1)
        cnt = torch.bincount(a, minlength=k)
        sums = torch.zeros_like(cent).index_add_(0, a, x)
        cent = torch.where((cnt > 0).unsqueeze(1), sums / cnt.clamp(min=1).unsqueeze(1), cent)
    return cent


class IvfPqIndex(IvfFlatIndex):
    """IVF-PQ (index_factory.cc:40-50 'ivfpq' / 'gpu_ivfpq', ``IndexOption.m`` sub-quantisers of 8 bits): the coarse
    quantiser and inverted lists of :class:`IvfFlatIndex`; every row is stored as ``m`` bytes - the nearest of 256
    codewords per sub-space of its residual to the list centroid.  A search scores rows by asymmetric distance
    computation (query-side look-up table, one table per (query, list)), keeps ``refine * k`` candidates and re-ranks
    them with the exact rows (``refine = 0``: return the quantised scores like a plain faiss IndexIVFPQ)."""

    def __init__(self, table, x: torch.Tensor, dim: int, nlist: int, nprobe: int, metric: int, m: int = 0, iters: int = 8,
                 seed: int = 0, refine: int = 4):
        super().__init__(table, x, dim, nlist, nprobe, metric, iters=iters, seed=seed)
        n = x.size(0)
        m = int(m) if m else max(1, min(64, dim // 4))
        self.m = max(1, min(m, dim, 128))
        self.dsub = (dim + self.m - 1) // self.m
        self.dimp = self.m * self.dsub                                  # dim padded to a multiple of m
        self.refine = int(refine)
        g = torch.Generator(device=x.device).manual_seed(seed + 1)
        cent = self._pad(self.centroids)
        self.centroids_p = cent.contiguous()
        # assignment of every row (list order is a stable sort of it): recover it from the offsets
        assign_sorted = torch.repeat_interleave(torch.arange(self.nlist, device=x.device), self.offsets[1:] - self.offsets[:-1])
        # residuals in LIST ORDER, chunked
        books = torch.zeros(self.m, 256, self.dsub, device=x.device)
        n_train = min(n, 256 * 64)
        if n > 0:
            tp = torch.randperm(n, device=x.device, generator=g)[:n_train]
            tr = self._pad(x[self.order[tp], :dim].float()) - cent[assign_sorted[tp]]
            for j in range(self.m):
                books[j] = _kmeans(tr[:, j * self.dsub:(j + 1) * self.dsub].contiguous(), 256, iters, g)
        self.codebooks = books.contiguous()
        codes = torch.empty(n, self.m, dtype=torch.uint8, device=x.device)
        for s in range(0, n, 1 << 16):
            pos = slice(s, min(n, s + (1 << 16)))
            r = self._pad(x[self.order[pos], :dim].float()) - cent[assign_sorted[pos]]
            for j in range(self.m):
                codes[pos, j] = torch.cdist(r[:, j * self.dsub:(j + 1) * self.dsub], books[j]).argmin(1).to(torch.uint8)
        self.codes = codes.contiguous()

    def _pad(self, v: torch.Tensor) -> torch.Tensor:
        if v.size(1) == self.dimp:
            return v
        return torch.cat([v, torch.zeros(v.size(0), self.dimp - v.size(1), device=v.device, dtype=v.dtype)], 1)

    def code_bytes(self) -> int:
        return int(self.codes.numel())

    def _adc_portable(self, q: torch.Tensor, probes: torch.Tensor, kk: int):
        """torch oracle of the scan kernel: same tables, same codes."""
        B = q.size(0)
        best_s = torch.full((B, kk), float("-inf"), device=q.device)
        best_i = torch.full((B, kk), -1, dtype=torch.int64, device=q.device)
        offs = self.offsets.tolist()
        ar = torch.arange(self.m, device=q.device)
        for b in range(B):
            cs, ci = [best_s[b]], [best_i[b]]
            for l in probes[b].tolist():
                lo, hi = offs[l], offs[l + 1]
                if hi == lo:
                    continue
                if self.metric == 1:
                    r = q[b].view(self.m, 1, self.dsub)
                    lut = (r * self.codebooks).sum(2)                                      # [m, 256]
                    bias = (q[b] * self.centroids_p[l]).sum()
                else:
                    r = (q[b] - self.centroids_p[l]).view(self.m, 1, self.dsub)
                    lut = -((r - self.codebooks) ** 2).sum(2)
                    bias = 0.0
                sc = lut[ar[None, :], self.codes[lo:hi].long()].sum(1) + bias
                cs.append(sc); ci.append(self.order[lo:hi])
            cs, ci = torch.cat(cs), torch.cat(ci)
            v, j = torch.topk(cs, min(kk, cs.numel()))
            best_s[b, :v.numel()], best_i[b, :v.numel()] = v, ci[j]
        best_i = torch.where(torch.isinf(best_s), torch.full_like(best_i, -1), best_i)
        return best_s, best_i

    def search(self, q: torch.Tensor, k: int, use_kernel: bool):
        qf = q.float()
        probes = torch.cdist(qf, self.centroids).topk(self.nprobe, dim=1, largest=False).indices.contiguous()
        qp = self._pad(qf).contiguous()
        kk = k if self.refine <= 0 else min(64, max(k, self.refine * k))
        if use_kernel and kk <= 64:
            from ..parallel.runtime import native
            s, r = native().knn_ivfpq_search(self.codes, self.order, self.offsets, qp, probes, self.centroids_p, self.codebooks,
                                             int(kk), int(self.metric))
            s = torch.where(r >= 0, s, torch.full_like(s, float("-inf")))
        else:
            s, r = self._adc_portable(qp, probes, kk)
        if self.refine <= 0:
            return s, r
        # exact re-rank of the kk candidates
        ok = r >= 0
        xr = self.x[r.clamp(min=0), :self.dim].float()                                     # [B, kk, d]
        ip = torch.einsum("bd,bkd->bk", qf, xr)
        sc = ip if self.metric == 1 else -((qf ** 2).sum(1, keepdim=True) - 2 * ip + (xr ** 2).sum(2))
        sc = torch.where(ok, sc, torch.full_like(sc, float("-inf")))
        v, j = torch.topk(sc, min(k, kk), dim=1)
        rows = torch.gather(r, 1, j)
        rows = torch.where(torch.isinf(v), torch.full_like(rows, -1), rows)
        return v, rows


def build_index(table, option) -> None:
    """``g.node(..., option=gl.IndexOption())``: attach the requested index to the node table
    (graphlearn/src/contrib/knn/builder.cc:23-52, local_noder.cc:44-51)."""
    itype = getattr(option, "index_type", "flat") or "flat"
    itype = itype.replace("gpu_", "")
    table._knn_option = (itype, int(getattr(option, "nlist", 0) or 0), int(getattr(option, "nprobe", 0) or 0),
                         int(getattr(option, "m", 0) or 0))
    table._knn_index = None


def search(rt, table, queries: torch.Tensor, k: int, metric: int = 0):
    """-> (ids [B, k], distances [B, k]); distances are squared L2 (metric 0) or inner products (1)."""
    W = rt.world
    q = queries.to(rt.device).float()
    dim = table.float_dim
    x_full = table.feats.local
    x = x_full[:, :dim]
    kern = _use_kernel(rt, x) and k <= 64
    itype, nlist, nprobe, pq_m = (tuple(getattr(table, "_knn_option", ("flat", 0, 0, 0))) + (0,))[:4]
    if itype in ("ivfflat", "ivfpq"):
        idx = getattr(table, "_knn_index", None)
        if idx is None or idx.x.data_ptr() != x_full.data_ptr() or idx.metric != metric:
            nl = nlist or max(1, int(x.size(0) ** 0.5))
            if itype == "ivfpq" and x_full.dtype in (torch.float32, torch.bfloat16):
                idx = IvfPqIndex(table, x_full, dim, nl, nprobe, metric, m=pq_m)
            else:
                idx = IvfFlatIndex(table, x_full, dim, nl, nprobe, metric)
            table._knn_index = idx
        s, rows = idx.search(q, k, kern)
    elif kern:
        s, rows = _kernel_topk(table, x_full, dim, q, k, metric)
    else:
        s, rows = _shard_topk(x, q, k, metric)
    if W > 1 and kern:
        # peer-memory merge: lists go into symmetric buffers, every rank reads all of them over NVLink
        from ..parallel.runtime import native
        B = q.size(0)
        key = ("knn_merge", B, k)
        bufs = rt.__dict__.setdefault("_knn_bufs", {})
        if key not in bufs:
            bufs[key] = (rt.symm_empty((B * k,), torch.float32), rt.symm_empty((B * k,), torch.int64))
        bs, bi = bufs[key]
        rt.barrier()                                    # previous readers are done with the buffers
        bs.local.copy_(s.reshape(-1)); bi.local.copy_(rows.reshape(-1))
        torch.cuda.synchronize()
        rt.barrier()
        ptrs = torch.tensor(list(bs.ptrs) + list(bi.ptrs), dtype=torch.int64)
        s, vids = native().knn_merge_peers(ptrs, W, B, k, s)
    else:
        vids = torch.where(rows >= 0, rows * W + rt.rank, rows)
        if W > 1:
            all_s = [torch.empty_like(s) for _ in range(W)]
            all_v = [torch.empty_like(vids) for _ in range(W)]
            dist.all_gather(all_s, s.contiguous())
            dist.all_gather(all_v, vids.contiguous())
            s, vids = torch.cat(all_s, 1), torch.cat(all_v, 1)
            s, j = torch.topk(s, k, dim=1)
            vids = torch.gather(vids, 1, j)
    ids = table.idmap.to_id(vids)
    d = s if metric == 1 else -s
    return ids, d


class KnnOperator(object):
    """Imperative form of ``Graph.search`` (graphlearn/python/operator/knn_operator.py): bound to a node type,
    ``search(inputs, k)`` returns (ids [B, k], distances [B, k]) as numpy arrays."""

    def __init__(self, graph, node_type):
        self._g, self._type = graph, node_type

    def search(self, inputs, k=1):
        return self._g.search(self._type, inputs, KnnOption(k))
