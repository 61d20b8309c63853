"""Per-GPU graph shards: node tables and CSR adjacency in HBM.

H100-native replacement for the reference's GraphStore / Graph / Noder and the
memory storages (graphlearn/src/core/graph/graph_store.cc:185-333,
storage/memory_adj_matrix.cc:159-225, memory_node_storage.cc:64-138):

* a node type is hash partitioned by ``|id| % world`` (hash_partitioner.h:90-92);
  local rows are addressed by *virtual ids* ``vid = row * world + owner`` so
  that any rank can compute (owner, row) arithmetically.  For a dense id space
  0..N-1 the vid is the id itself (row = id // world).
* float attributes live in ONE symmetric [n_local, stride] table (fp32 or bf16)
  that every peer maps over NVLink; labels / weights / int attrs are local
  device tensors (also published symmetrically for remote lookups).
* an edge type is a CSR over the source rows, stored on the source's owner:
  ``indptr`` int64, ``indices`` = destination vids, optional in-row inclusive
  prefix sums of the sampling weights (weighted sampling without per-call alias
  builds, SURVEY 7.4 item 5) and optional timestamps (rows sorted ascending for
  temporal graphs, otherwise by weight descending so that top-k is a prefix -
  memory_adj_matrix.cc:60-66,105-149).  The edge id is the CSR position on the
  owner, so no separate eid array is needed.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch

from .. import config as _config
from ..parallel import partition as part
from ..parallel.runtime import Runtime, SymmTensor, make_csr_desc, make_table_desc


def _round_up(x, m):
    return (x + m - 1) // m * m


def sorted_unique(ids: torch.Tensor) -> torch.Tensor:
    """``torch.unique(ids)`` (sorted) without the sort when the id space is reasonably dense: a presence bitmap
    + ``nonzero`` is O(n) and ~5x faster on 10^8 edge end points (the sort-based unique dominated the CPU build)."""
    n = int(ids.numel())
    if n < (1 << 20):
        return torch.unique(ids)
    lo, hi = int(ids.min().item()), int(ids.max().item())
    if lo < 0 or hi >= 8 * n:
        return torch.unique(ids)
    present = torch.zeros(hi + 1, dtype=torch.bool, device=ids.device)
    present[ids] = True
    return present.nonzero().flatten()


class IdMap:
    """global id <-> vid for one node type."""

    def __init__(self, rt: Runtime, local_ids: torch.Tensor, dense: bool):
        self.rt = rt
        self.dense = dense
        self.local_ids = local_ids              # sorted ascending (general) / implicit (dense)
        self.n_local = int(local_ids.numel())
        self.nrows = rt.all_gather_object(self.n_local)
        # non-dense id spaces on CUDA: the sorted ids live in a symmetric buffer so that ANY rank translates
        # id <-> vid with a peer-memory binary search (csrc/idmap.cu) - no collective, no lock-step epochs
        self.peer_desc = None
        if not dense and rt.is_cuda:
            st = rt.symm_empty((max(self.n_local, 1),), torch.int64)
            if self.n_local:
                st.local[:self.n_local].copy_(local_ids)
            self._symm_ids = st
            pad = lambda xs: list(xs) + [0] * (8 - len(xs))  # noqa: E731
            self.peer_desc = torch.tensor([rt.world] + pad(self.nrows) + pad(st.ptrs), dtype=torch.int64)
            rt.barrier()

    @property
    def collective(self) -> bool:
        """True when to_vid / to_id are collectives (every rank must call them together)."""
        return (not self.dense) and self.rt.world > 1 and self.peer_desc is None

    @staticmethod
    def build(rt: Runtime, local_ids: torch.Tensor) -> "IdMap":
        """`local_ids`: unique ids owned by this rank (any order)."""
        local_ids = sorted_unique(local_ids)
        n = int(local_ids.numel())
        W = rt.world
        # dense iff the owned ids are exactly {rank, rank+W, rank+2W, ...}
        dense_local = bool(n == 0 or (int(local_ids[0]) == rt.rank and int(local_ids[-1]) == rt.rank + (n - 1) * W)) \
            and bool(n == 0 or torch.equal(local_ids, torch.arange(n, device=local_ids.device) * W + rt.rank))
        dense = all(rt.all_gather_object(dense_local))
        return IdMap(rt, local_ids, dense)

    def _local_rows(self, ids: torch.Tensor) -> torch.Tensor:
        """rows of ids owned by THIS rank; -1 when unknown."""
        W = self.rt.world
        if self.dense:
            rows = torch.div(ids, W, rounding_mode="floor")
            ok = (ids >= 0) & (rows < self.n_local) & (ids % W == self.rt.rank)
            return torch.where(ok, rows, torch.full_like(rows, -1))
        if self.n_local == 0:
            return torch.full_like(ids, -1)
        pos = torch.searchsorted(self.local_ids, ids).clamp_(max=self.n_local - 1)
        ok = self.local_ids[pos] == ids
        return torch.where(ok, pos, torch.full_like(pos, -1))

    def to_vid(self, ids: torch.Tensor) -> torch.Tensor:
        """Collective when world > 1 and the id space is not dense."""
        W = self.rt.world
        ids = ids.to(torch.int64)
        if self.dense:
            rows = torch.div(ids, W, rounding_mode="floor")
            nrows = torch.tensor(self.nrows, device=ids.device, dtype=torch.int64)
            ok = (ids >= 0) & (rows < nrows[(ids.abs() % W)])
            return torch.where(ok, ids, torch.full_like(ids, -1))
        if W == 1:
            return self._local_rows(ids)        # vid == row
        if self.peer_desc is not None and ids.is_cuda:
            from ..parallel.runtime import native
            return native().idmap_translate(self.peer_desc, ids.reshape(-1), True).reshape(ids.shape)
        flat = ids.reshape(-1)
        (rows,) = part.remote_apply(flat, lambda x: (self._local_rows(x),), W)
        vid = torch.where(rows >= 0, rows * W + part.owner_of(flat, W), torch.full_like(rows, -1))
        return vid.reshape(ids.shape)

    def local_vids(self) -> torch.Tensor:
        W = self.rt.world
        return torch.arange(self.n_local, device=self.local_ids.device, dtype=torch.int64) * W + self.rt.rank

    def to_id(self, vids: torch.Tensor) -> torch.Tensor:
        """vid -> original id (collective when not dense and world > 1)."""
        if self.dense:
            return vids
        W = self.rt.world
        flat = vids.reshape(-1)

        def look(v):
            rows = torch.div(v, W, rounding_mode="floor").clamp_(min=0, max=max(self.n_local - 1, 0))
            out = self.local_ids[rows] if self.n_local > 0 else torch.full_like(v, -1)
            return (torch.where(v >= 0, out, torch.full_like(out, -1)),)

        if W == 1:
            return look(flat)[0].reshape(vids.shape)
        if self.peer_desc is not None and vids.is_cuda:
            from ..parallel.runtime import native
            return native().idmap_translate(self.peer_desc, flat, False).reshape(vids.shape)
        # route by owner = vid % W (vids are non-negative when valid)
        (ids,) = part.remote_apply(flat.clamp(min=0), look, W)
        return torch.where(flat >= 0, ids, torch.full_like(ids, -1)).reshape(vids.shape)


class _NoCache(object):
    """view of a SymmTensor that hides its replica cache (used while filling the cache)."""

    def __init__(self, st):
        self.local, self.nrows, self.ptrs = st.local, st.nrows, st.ptrs
        self.cache_map = self.cache_rows = None


class NodeTable:
    def __init__(self, rt: Runtime, ntype: str, idmap: IdMap):
        self.rt = rt
        self.type = ntype
        self.idmap = idmap
        self.n_local = idmap.n_local
        self.float_dim = 0
        self.int_dim = 0
        self.str_dim = 0
        self.feats: Optional[SymmTensor] = None      # [n_local, stride]
        self.feat_desc: Optional[torch.Tensor] = None
        self.ints: Optional[SymmTensor] = None       # int64 [n_local, int_dim]
        self.labels: Optional[SymmTensor] = None     # int64 [n_local]
        self.weights: Optional[SymmTensor] = None    # float [n_local]
        self.timestamps: Optional[SymmTensor] = None
        self.strings: Optional[List[List[str]]] = None   # host side, [n_local][str_dim]
        self.out_degrees: Dict[str, torch.Tensor] = {}
        self.in_degrees: Dict[str, torch.Tensor] = {}
        self.present: Optional[torch.Tensor] = None  # bool [n_local]: row came from a node source

    @property
    def nrows(self):
        return self.idmap.nrows

    FP8_BLOCK = 32

    @staticmethod
    def quantize_fp8_rows(x: torch.Tensor, stride: int) -> torch.Tensor:
        """fp32 [n, d] -> uint8 [n, stride] rows ``[d e4m3 bytes | pad to 16][one bf16 scale per 32 elements][pad]`` with
        value = q * scale and scale = bf16(amax(block) / 448) (448 = largest e4m3 magnitude)."""
        n, d = int(x.size(0)), int(x.size(1))
        B = NodeTable.FP8_BLOCK
        nb = (d + B - 1) // B
        xp = torch.zeros(n, nb * B, dtype=torch.float32, device=x.device)
        xp[:, :d] = x.float()
        blocks = xp.view(n, nb, B)
        scale = (blocks.abs().amax(2) / 448.0).to(torch.bfloat16)
        scale = torch.where(scale.float() > 0, scale, torch.ones_like(scale))
        # the bf16 rounding of the scale may push |x / scale| just above 448: clamp before the cast (e4m3fn has no inf)
        q = (blocks / scale.float().unsqueeze(2)).clamp_(-448.0, 448.0).to(torch.float8_e4m3fn)
        out = torch.zeros(n, stride, dtype=torch.uint8, device=x.device)
        out[:, :d] = q.view(n, nb * B)[:, :d].view(torch.uint8)
        soff = _round_up(d, 16)
        out[:, soff:soff + 2 * nb] = scale.contiguous().view(torch.uint8).view(n, 2 * nb)
        return out

    @staticmethod
    def dequantize_fp8_rows(t: torch.Tensor, d: int) -> torch.Tensor:
        """uint8 [n, stride] fp8 rows -> fp32 [n, d]"""
        B = NodeTable.FP8_BLOCK
        nb = (d + B - 1) // B
        soff = _round_up(d, 16)
        q = t[:, :d].contiguous().view(torch.float8_e4m3fn).float()
        scale = t[:, soff:soff + 2 * nb].contiguous().view(torch.bfloat16).float()
        return q * scale.repeat_interleave(B, dim=1)[:, :d]

    def dequantize_local(self, rows: Optional[torch.Tensor] = None) -> torch.Tensor:
        """fp32 values of (a subset of) the local rows of an fp8 table - oracle / portable path"""
        return NodeTable.dequantize_fp8_rows(self.feats.local if rows is None else self.feats.local[rows], self.float_dim)

    def set_float(self, x: torch.Tensor, dtype: torch.dtype = torch.float32):
        """x: [n_local, d] on the runtime device.  dtype: torch.float32 / torch.bfloat16 / torch.float8_e4m3fn (block-scaled
        fp8 storage: half the bytes of bf16 - read by the fused layer kernel and by lookups, dequantised on the fly)."""
        d = int(x.size(1))
        self.float_dim = d
        if dtype == torch.float8_e4m3fn:
            nb = (d + NodeTable.FP8_BLOCK - 1) // NodeTable.FP8_BLOCK
            stride = _round_up(_round_up(d, 16) + 2 * nb, 16)
            align = int(getattr(_config.get(), "feature_row_align", 128))
            if align > 16 and stride > align // 2:
                stride = _round_up(stride, align)
            st = self.rt.symm_empty((self.n_local, stride), torch.uint8)
            st.local.copy_(NodeTable.quantize_fp8_rows(x, stride))
            self.feats = st
            self.rt.barrier()
            self.feat_desc = make_table_desc(self.rt.world, d, stride, torch.float8_e4m3fn, st.nrows, st.ptrs)
            return
        esz = 4 if dtype == torch.float32 else 2
        stride = _round_up(max(d, 1), 16 // esz)
        # rows wider than one 128-byte line start on a line boundary: a 200-byte row then touches exactly 2 lines instead
        # of 2.6 on average - over NVLink (whole lines travel) that is 23 % fewer bytes, and HBM has room for the padding.
        # `config.feature_row_align` = 16 restores dense rows.
        align = int(getattr(_config.get(), "feature_row_align", 128))
        if align > 16 and d * esz > align // 2:
            stride = _round_up(d * esz, align) // esz
        st = self.rt.symm_empty((self.n_local, stride), dtype)
        st.local.zero_()
        st.local[:, :d] = x.to(dtype)
        self.feats = st
        self.rt.barrier()
        self.feat_desc = make_table_desc(self.rt.world, d, stride, dtype, st.nrows, st.ptrs)

    # ------------------------------------------------------------------ N17: replica cache of remote rows
    def build_feature_cache(self, capacity: int, scores: Optional[torch.Tensor] = None) -> int:
        """Replicate up to ``capacity`` REMOTE float-feature rows into this rank's HBM.

        Reference: the optional LFU cache of remote node attributes
        (graphlearn/src/core/graph/storage/remote_node_storage.cc:55-82, cache_policy.h:37-78,
        enabled by ``set_local_node_cache_capacity``).  GPU design: a STATIC, score-ordered
        replica (highest global in-degree first, PaGraph style) because a device kernel cannot
        maintain LFU state cheaply and 180 GB of HBM usually holds the whole table; the kernels
        resolve ``vid -> cache slot`` through one int32 map (csrc/host_utils.h TableView).
        ``scores``: float/int tensor indexed by vid (higher = hotter), identical on every rank;
        None = cache in vid order.  Collective.  Returns the number of cached rows."""
        rt, W = self.rt, self.rt.world
        if W == 1 or self.feats is None or capacity <= 0:
            return 0
        if self.feats.local.dtype == torch.uint8:
            raise NotImplementedError("the replica cache copies rows through the float gather: not wired for fp8 tables yet")
        dev = rt.device
        max_vid = max(int(n) for n in self.nrows) * W
        vid = torch.arange(max_vid, device=dev, dtype=torch.int64)
        nrows = torch.tensor([int(n) for n in self.nrows], device=dev, dtype=torch.int64)
        exists = torch.div(vid, W, rounding_mode="floor") < nrows[vid % W]
        remote = exists & ((vid % W) != rt.rank)
        n_remote = int(remote.sum().item())
        C = min(int(capacity), n_remote)
        if C <= 0:
            return 0
        if C == n_remote:
            sel = vid[remote]
        else:
            sc = torch.zeros(max_vid, device=dev, dtype=torch.float32) if scores is None else \
                scores.to(dev).float()[:max_vid].clone()
            if scores is None:
                sc = -vid.float()
            sc[~remote] = float("-inf")
            sel = torch.topk(sc, C).indices.sort().values
        st = self.feats
        stride = int(st.local.size(1))
        rows = torch.zeros(C, stride, dtype=st.local.dtype, device=dev)
        from ..ops import gather as G
        base_desc = make_table_desc(W, self.float_dim, stride, st.local.dtype, st.nrows, st.ptrs) \
            if rt.is_cuda else None
        step = 1 << 20
        # every rank must run the same number of (collective on the portable path) rounds
        n_rounds = (max(rt.all_gather_object(C)) + step - 1) // step
        for i in range(n_rounds):
            chunk = sel[i * step:(i + 1) * step]
            got = G.gather_rows(rt, _NoCache(st), base_desc, chunk, self.float_dim, out_dtype=st.local.dtype)
            if chunk.numel():
                rows[i * step:i * step + chunk.numel(), :self.float_dim] = got
        cmap = torch.full((max_vid,), -1, dtype=torch.int32, device=dev)
        cmap[sel] = torch.arange(C, device=dev, dtype=torch.int32)
        st.cache_map, st.cache_rows = cmap, rows
        rt.barrier()
        if rt.is_cuda:
            if C == n_remote:
                # FULL replica: `sel` is sorted by vid, so the rows of owner r form the strided subsequence
                # vid % W == r in row order.  Regroup them per owner and point the descriptor's peer slot r
                # at the local copy: kernels then run the plain local path (no map lookup at all).
                owner = sel % W
                ptrs, keep = list(st.ptrs), []
                for r in range(W):
                    if r == rt.rank:
                        continue
                    rep = rows[owner == r].contiguous()          # [nrows[r], stride], row order == owner's
                    assert rep.size(0) == int(self.nrows[r])
                    keep.append(rep)
                    ptrs[r] = rep.data_ptr()
                st.replicas = keep
                st.cache_map = st.cache_rows = None       # the regrouped copies replace the slot table
                self.feat_desc = make_table_desc(W, self.float_dim, stride, st.local.dtype, st.nrows, ptrs)
            else:
                self.feat_desc = make_table_desc(W, self.float_dim, stride, st.local.dtype, st.nrows, st.ptrs,
                                                 cache=(rt.rank, cmap.data_ptr(), rows.data_ptr()))
        return C

    # ---- LFU policy (reference: cache_policy.h:37-78 LFU over node ids, remote_node_storage.cc:55-82)
    # A device kernel cannot keep per-access LFU lists, but the engine knows every row it is about to read: the sampled
    # hop ids.  ``observe_access`` adds them to a per-vid frequency table (one histogram kernel over ids that are already
    # on the device), ``refresh_feature_cache_lfu`` re-selects the ``capacity`` most frequently read REMOTE rows and
    # rebuilds the replica - i.e. LFU with batched (epoch / every-N-steps) eviction instead of per-access eviction.
    def observe_access(self, vids: torch.Tensor):
        W = self.rt.world
        max_vid = max(int(n) for n in self.nrows) * W
        if getattr(self, "_lfu_freq", None) is None or self._lfu_freq.numel() != max_vid:
            self._lfu_freq = torch.zeros(max_vid, dtype=torch.float32, device=self.rt.device)
        v = vids.reshape(-1)
        v = v[(v >= 0) & (v < max_vid)]
        if v.numel():
            self._lfu_freq.index_add_(0, v, torch.ones(v.numel(), dtype=torch.float32, device=v.device))

    def refresh_feature_cache_lfu(self, capacity: int, decay: float = 0.5) -> int:
        """Rebuild the replica cache from the access frequencies seen so far (collective); old counts decay so the
        policy follows a drifting workload."""
        freq = getattr(self, "_lfu_freq", None)
        self.drop_feature_cache()
        n = self.build_feature_cache(capacity, scores=freq)
        if freq is not None:
            freq.mul_(decay)
        return n

    def drop_feature_cache(self):
        st = self.feats
        if st is None or (getattr(st, "cache_map", None) is None and getattr(st, "replicas", None) is None):
            return
        st.cache_map = st.cache_rows = None
        st.replicas = None
        if self.rt.is_cuda:
            self.feat_desc = make_table_desc(self.rt.world, self.float_dim, int(st.local.size(1)), st.local.dtype,
                                             st.nrows, st.ptrs)

    def lookup_strings(self, vids: torch.Tensor, default: str = ""):
        """[n, str_dim] object array of the string attributes of `vids`.  Strings live on the HOST of the owning
        rank: one rank = direct indexing; several ranks = request / response exchange of pickled lists (two
        ``all_gather_object`` rounds - the reference ships strings inside its LookupNodes protobuf responses).
        Collective when world > 1."""
        import numpy as np
        W, r = self.rt.world, self.rt.rank
        v = vids.reshape(-1).cpu().numpy()

        def local_rows(req):
            rows = req // W
            out = np.full((len(req), self.str_dim), default, dtype=object)
            if self.strings is not None:
                ok = (req >= 0) & (rows < self.n_local)
                if ok.any():
                    out[ok] = self.strings[rows[ok]]
            return out

        if W == 1:
            return local_rows(v)
        arr = np.full((len(v), self.str_dim), default, dtype=object)
        owner = np.where(v >= 0, v % W, -1)
        asked = self.rt.all_gather_object([v[owner == o] for o in range(W)])   # asked[q][o]: rank q wants from rank o
        got = self.rt.all_gather_object([local_rows(np.asarray(asked[q][r], dtype=np.int64)) for q in range(W)])
        for o in range(W):
            m = owner == o
            if m.any():
                arr[m] = got[o][r]
        return arr

    def _set_symm(self, name, x: torch.Tensor):
        st = self.rt.symm_empty(tuple(x.shape), x.dtype)
        st.local.copy_(x)
        setattr(self, name, st)
        self.rt.barrier()

    def set_labels(self, x):
        self._set_symm("labels", x.to(torch.int64))

    def set_weights(self, x):
        self._set_symm("weights", x.to(torch.float32))

    def set_timestamps(self, x):
        self._set_symm("timestamps", x.to(torch.int64))

    def set_ints(self, x):
        self.int_dim = int(x.size(1))
        self._set_symm("ints", x.to(torch.int64))


class CsrShard:
    """CSR adjacency of one edge type on this rank (+ peer pointer tables)."""

    def __init__(self, rt: Runtime, etype: str, src_type: str, dst_type: str):
        self.rt = rt
        self.type = etype
        self.src_type = src_type
        self.dst_type = dst_type
        self.indptr: Optional[SymmTensor] = None
        self.indices: Optional[SymmTensor] = None
        self.cumw: Optional[SymmTensor] = None          # edge-weight prefix sums
        self.cumw_indeg: Optional[SymmTensor] = None    # in-degree prefix sums
        self.ts: Optional[SymmTensor] = None
        self.weights: Optional[SymmTensor] = None       # float [E_local]
        self.labels: Optional[SymmTensor] = None
        self.float_attrs: Optional[SymmTensor] = None
        self.int_attrs: Optional[SymmTensor] = None
        self.float_dim = 0
        self.int_dim = 0
        self.n_src_rows = 0
        self.n_edges = 0
        self.desc: Optional[torch.Tensor] = None
        self.desc_indeg: Optional[torch.Tensor] = None
        self.directed = True
        self.timestamped = False
        self.dst_ids_unique: Optional[torch.Tensor] = None   # distinct dst vids on this shard (neg sampling)

    def insertion_pos(self) -> torch.Tensor:
        """CSR position of the i-th INSERTED edge of this shard (inverse of ``_order``)."""
        if getattr(self, "_ins_pos", None) is None:
            inv = torch.empty_like(self._order)
            inv[self._order] = torch.arange(self._order.numel(), device=self._order.device)
            self._ins_pos = inv
        return self._ins_pos

    @staticmethod
    def from_coo(rt: Runtime, etype, src_type, dst_type, src_rows: torch.Tensor, dst_vids: torch.Tensor,
                 n_src_rows: int, weights: Optional[torch.Tensor] = None, ts: Optional[torch.Tensor] = None,
                 labels: Optional[torch.Tensor] = None, float_attrs: Optional[torch.Tensor] = None,
                 int_attrs: Optional[torch.Tensor] = None, eids: Optional[torch.Tensor] = None) -> "CsrShard":
        """K11: build the CSR on the device.  Rows are ordered by timestamp
        ascending when `ts` is given, else by weight descending (top-k prefix)."""
        self = CsrShard(rt, etype, src_type, dst_type)
        E = int(src_rows.numel())
        dev = src_rows.device
        order = torch.arange(E, device=dev)
        indptr = None
        grouped = E > 0 and ts is None and weights is None and bool((src_rows[1:] >= src_rows[:-1]).all())
        if E > 0 and not grouped and dev.type == "cuda" and _config.get().native_csr_build:
            # counting build (csrc/csr_build.cu): histogram -> prefix sum -> scatter -> per-row sort; the same permutation
            # as the two stable sorts below, without sorting E keys globally
            from ..parallel.runtime import native
            if ts is not None:
                indptr, order = native().csr_build(src_rows.to(torch.int64).contiguous(), n_src_rows, ts.to(torch.int64), 1)
            elif weights is not None:
                indptr, order = native().csr_build(src_rows.to(torch.int64).contiguous(), n_src_rows, weights.to(torch.float32), 2)
            else:
                indptr, order = native().csr_build(src_rows.to(torch.int64).contiguous(), n_src_rows, None, 0)
        elif E > 0 and not grouped:
            if ts is not None:
                order = torch.argsort(ts, stable=True)
            elif weights is not None:
                order = torch.argsort(weights, descending=True, stable=True)
            order = order[torch.argsort(src_rows[order], stable=True)]
        srt = src_rows[order]
        if indptr is None:
            counts = torch.bincount(srt, minlength=n_src_rows) if E > 0 else torch.zeros(n_src_rows, dtype=torch.int64, device=dev)
            indptr = torch.zeros(n_src_rows + 1, dtype=torch.int64, device=dev)
            indptr[1:] = torch.cumsum(counts, 0)
        self.n_src_rows = n_src_rows
        self.n_edges = E
        self.indptr = rt.symm_from(indptr)
        self.indices = rt.symm_from(dst_vids[order].to(torch.int64))
        self._order = order
        self._row_of_edge = srt
        if weights is not None:
            w = weights[order].to(torch.float32)
            self.weights = rt.symm_from(w)
            self.cumw = rt.symm_from(self._row_cumsum(w, indptr, srt))
        if ts is not None:
            self.ts = rt.symm_from(ts[order].to(torch.int64))
            self.timestamped = True
        if eids is not None:       # explicit edge ids (in-edge CSR: position of the edge in the forward CSR)
            self.eids = rt.symm_from(eids[order].to(torch.int64))
        if labels is not None:
            self.labels = rt.symm_from(labels[order].to(torch.int64))
        if float_attrs is not None and float_attrs.numel() > 0:
            self.float_dim = int(float_attrs.size(1))
            self.float_attrs = rt.symm_from(float_attrs[order].to(torch.float32))
        if int_attrs is not None and int_attrs.numel() > 0:
            self.int_dim = int(int_attrs.size(1))
            self.int_attrs = rt.symm_from(int_attrs[order].to(torch.int64))
        self.dst_ids_unique = sorted_unique(self.indices.local) if E > 0 else torch.zeros(0, dtype=torch.int64, device=dev)
        self._make_desc()
        return self

    @staticmethod
    def _row_cumsum(w: torch.Tensor, indptr: torch.Tensor, row_of_edge: torch.Tensor) -> torch.Tensor:
        if w.numel() == 0:
            return w.clone()
        c = torch.cumsum(w.to(torch.float64), 0)
        base = torch.zeros(indptr.numel() - 1, dtype=torch.float64, device=w.device)
        starts = indptr[:-1]
        nz = starts < w.numel()
        base[nz] = c[starts[nz]] - w[starts[nz]].to(torch.float64)
        return (c - base[row_of_edge]).to(torch.float32)

    def set_indegree_weights(self, indeg_of_dst: torch.Tensor):
        """per-edge weight = in-degree of the destination (InDegreeSampler)."""
        w = indeg_of_dst.to(torch.float32).clamp_(min=0)
        self.cumw_indeg = self.rt.symm_from(self._row_cumsum(w, self.indptr.local, self._row_of_edge))
        self._make_desc()

    def ensure_sorted_rows(self):
        """id-sorted copy of every adjacency row (same indptr), peer mapped: the walk kernel's node2vec membership test
        becomes a binary search.  Collective (symmetric allocation); built once, on first use."""
        if getattr(self, "sorted_idx", None) is None:
            idx = self.indices.local
            if idx.numel():
                key = self._row_of_edge * (int(idx.max().item()) + 2) + (idx + 1)       # (row, dst) lexicographic
                srt = idx[torch.argsort(key)]
            else:
                srt = idx.clone()
            self.sorted_idx = self.rt.symm_from(srt)
            self._make_desc()
        return self.sorted_idx

    def _make_desc(self):
        W = self.rt.world
        srt = getattr(self, "sorted_idx", None)
        self.desc = make_csr_desc(
            W, self.indptr.nrows and [n - 1 for n in self.indptr.nrows], self.indptr.ptrs, self.indices.ptrs,
            self.eids.ptrs if getattr(self, "eids", None) is not None else None,
            self.cumw.ptrs if self.cumw is not None else None,
            self.ts.ptrs if self.ts is not None else None,
            srt.ptrs if srt is not None else None)
        if self.cumw_indeg is not None:
            self.desc_indeg = make_csr_desc(
                W, [n - 1 for n in self.indptr.nrows], self.indptr.ptrs, self.indices.ptrs, None,
                self.cumw_indeg.ptrs, self.ts.ptrs if self.ts is not None else None)

    @property
    def peer_ok(self) -> bool:
        return self.rt.is_cuda
