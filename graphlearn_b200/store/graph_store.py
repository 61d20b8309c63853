"""GraphStore: load -> partition -> build the per-GPU shards of a heterogeneous graph.

H100-native counterpart of GraphStore::{Load,Build,BuildStatistics}
(graphlearn/src/core/graph/graph_store.cc:185-333) and of the server Init
sequence (graphlearn/src/service/server_impl.cc:163-195):

  load     native multi-threaded TSV parser (csrc/host_loader.cpp) or in-memory
           arrays -> columnar tensors
  shuffle  rows are assigned to owner = |id| % world (edges by SRC id, nodes by
           node id - graph_update_request.cc:151-156,234-237).  Every rank
           parses 1/world of each file (byte-range slices, or whole files of a
           directory dealt round-robin) and one all-to-all-v per column moves
           the rows to their owners (parallel/partition.py shuffle_rows).
  build    id maps (id <-> virtual id), node tables and CSR shards in HBM, peer
           pointer tables exchanged through CUDA IPC.
"""
from __future__ import annotations

import os
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .. import config as _config
from ..data.decoder import Decoder
from ..parallel import partition as part
from ..parallel.runtime import Runtime, native
from .shards import CsrShard, IdMap, NodeTable, sorted_unique

ORIGIN, REVERSED = 0, 1


class EdgeInfo(object):
    def __init__(self, src_type, dst_type):
        self.src_type, self.dst_type = src_type, dst_type


class Topology(object):
    """edge type -> (src type, dst type)  (graphlearn/python/data/topology.py)."""

    def get_edge_info(self, edge_type):
        if edge_type not in self._edges:
            raise ValueError("edge_type {} not exists in the graph.".format(edge_type))
        return EdgeInfo(*self._edges[edge_type])

    def print_all(self):
        for k, (s, d) in self._edges.items():
            print("edge_type:{}, src_type:{}, dst_type:{}\n".format(k, s, d))

    def print_one(self, edge_type):
        e = self.get_edge_info(edge_type)
        print("edge_type:{}, src_type:{}, dst_type:{}\n".format(edge_type, e.src_type, e.dst_type))

    def __init__(self):
        self._edges: Dict[str, Tuple[str, str]] = {}

    def add(self, edge_type, src_type, dst_type):
        self._edges[edge_type] = (src_type, dst_type)

    def get_src_type(self, edge_type):
        return self._edges[edge_type][0]

    def get_dst_type(self, edge_type):
        return self._edges[edge_type][1]

    def is_exist(self, edge_type):
        return edge_type in self._edges

    def edge_types(self):
        return list(self._edges)

    def __str__(self):
        return "\n".join("%s: %s -> %s" % (e, s, d) for e, (s, d) in self._edges.items())


class Source(object):
    def __init__(self, kind, path, types, decoder, direction=ORIGIN, option=None, data=None):
        self.kind = kind              # 'node' | 'edge'
        self.path = path
        self.types = types            # node type | (src_type, dst_type, edge_type)
        self.decoder = decoder
        self.direction = direction
        self.option = option
        self.data = data              # optional in-memory dict of arrays


def _expand_paths(path: str) -> List[str]:
    """comma list / directory / URL -> LOCAL file paths (remote objects are spooled, io/filesystem.py)"""
    from ..io import filesystem as _fs
    return [_fs.localize(p) for p in _fs.expand(path)]


def _loader_threads(ranks_on_box: int) -> int:
    n = int(_config.get().loader_threads)
    return n if n > 0 else max(1, (os.cpu_count() or 8) // max(int(ranks_on_box), 1))


def storage_kinds(dec: Decoder) -> List[str]:
    """per attribute position: the column group it is stored in ('int' | 'float' | 'string'; hashed strings are ints)"""
    out = []
    for name, bucket, multival in dec._parsed:
        out.append("int" if name == "int" or (name == "string" and bucket is not None and not multival) else name)
    return out


def _load_source(src: Source, part_index: int = 0, part_count: int = 1) -> Dict[str, object]:
    """``Graph.node_attributes / edge_attributes`` selections (``src.use_attrs``: attribute positions of the FULL decoder
    ``src.decoder_full``) are applied after parsing: the unselected columns are dropped here and never reach the device."""
    use = getattr(src, "use_attrs", None)
    if use is None:
        return _load_source_all(src, src.decoder, part_index, part_count)
    full: Decoder = src.decoder_full
    out = _load_source_all(src, full, part_index, part_count)
    kinds = storage_kinds(full)
    col = {}
    seen = {"int": 0, "float": 0, "string": 0}
    for i, k in enumerate(kinds):
        col[i] = seen[k]
        seen[k] += 1
    pick = {"int": [col[i] for i in use if kinds[i] == "int"], "float": [col[i] for i in use if kinds[i] == "float"],
            "string": [col[i] for i in use if kinds[i] == "string"]}
    if out["ia"] is not None:
        out["ia"] = out["ia"][:, pick["int"]] if pick["int"] else None
    if out["fa"] is not None:
        out["fa"] = out["fa"][:, pick["float"]] if pick["float"] else None
    if out["strs"] is not None:
        out["strs"] = np.asarray(out["strs"], dtype=object)[:, pick["string"]] if pick["string"] else None
    return out


def _load_source_all(src: Source, dec: Decoder, part_index: int = 0, part_count: int = 1) -> Dict[str, object]:
    """-> dict(a, b, w, label, ts, ia, fa, strs) of CPU tensors.

    ``part_count > 1`` reads only this rank's share (SliceReader, graphlearn/src/core/io/
    slice_reader.h:60-86,137-157): a single file is cut into ``part_count`` contiguous record
    ranges; the files of a directory are dealt round-robin, whole, to the parts."""
    if src.data is not None:
        d = src.data
        g = lambda k: (None if d.get(k) is None else torch.as_tensor(np.asarray(d[k]) if not isinstance(d[k], torch.Tensor) else d[k]))  # noqa: E731
        a = g("ids") if src.kind == "node" else g("src_ids")
        out = {"a": a.to(torch.int64), "b": None if src.kind == "node" else g("dst_ids").to(torch.int64),
               "w": g("weights"), "label": g("labels"), "ts": g("timestamps"), "ia": g("int_attrs"),
               "fa": g("float_attrs"), "strs": d.get("string_attrs")}
        return out
    C = native()
    cfg = _config.get()
    codes, buckets = dec.loader_schema()
    parts = []
    paths = _expand_paths(src.path)
    if not paths:
        raise FileNotFoundError("no data files for source %r" % (src.path,))
    for j, p in enumerate(paths):
        if len(paths) > 1 and part_count > 1:
            if j % part_count != part_index:
                continue
            pi, pc = 0, 1
        else:
            pi, pc = part_index, part_count
        parts.append(C.load_table(p, src.kind == "edge", dec.weighted, dec.labeled, dec.timestamped, codes, buckets,
                                  dec.attr_delimiter, cfg.field_delimiter, _loader_threads(part_count), pi, pc))
    if not parts:       # more ranks than files: this rank contributes an empty slice
        parts.append(C.load_table(paths[0], src.kind == "edge", dec.weighted, dec.labeled, dec.timestamped, codes,
                                  buckets, dec.attr_delimiter, cfg.field_delimiter, 1, 0, 1))
        parts[0] = [t[:0] if i < 7 else t for i, t in enumerate(parts[0])]
        parts[0][7] = parts[0][7][:0]
        parts[0][8] = parts[0][8][:1]
    cat = [torch.cat([p[i] for p in parts]) if i < 7 else None for i in range(7)]
    strs = None
    if dec.string_attr_num > 0:
        rows = []
        for p in parts:
            blob = p[7].numpy().tobytes()
            off = p[8].tolist()
            vals = [blob[off[i]:off[i + 1]].decode("utf-8", "replace") for i in range(len(off) - 1)]
            rows.extend(vals)
        strs = np.array(rows, dtype=object).reshape(-1, dec.string_attr_num)
    n = cat[0].numel()
    return {"a": cat[0], "b": cat[1] if src.kind == "edge" else None,
            "w": cat[2] if dec.weighted else None, "label": cat[3] if dec.labeled else None,
            "ts": cat[4] if dec.timestamped else None,
            "ia": cat[5].view(n, -1) if dec.int_attr_num > 0 else None,
            "fa": cat[6].view(n, -1) if dec.float_attr_num > 0 else None, "strs": strs}


def _take(d: Dict[str, object], idx: torch.Tensor) -> Dict[str, object]:
    out = {}
    for k, v in d.items():
        if v is None:
            out[k] = None
        elif isinstance(v, torch.Tensor):
            out[k] = v[idx]
        else:
            out[k] = v[idx.numpy()]
    return out


class GraphStore(object):
    def __init__(self, rt: Runtime):
        self.rt = rt
        self.topology = Topology()
        self.node_decoders: Dict[str, Decoder] = {}
        self.edge_decoders: Dict[str, Decoder] = {}
        self.nodes: Dict[str, NodeTable] = {}
        self.edges: Dict[str, CsrShard] = {}
        self.reverse: Dict[str, CsrShard] = {}      # in-edge CSR (built lazily for inV / in-degree)
        self._edge_cache: Dict[str, Dict[str, torch.Tensor]] = {}
        self.stats: Dict[str, List[int]] = {}

    # ------------------------------------------------------------------ build
    def build(self, node_sources: List[Source], edge_sources: List[Source]):
        rt, W, r = self.rt, self.rt.world, self.rt.rank
        dev = rt.device
        cfg = _config.get()
        fdt = {"bf16": torch.bfloat16, "fp8": torch.float8_e4m3fn}.get(cfg.feature_dtype, torch.float32)
        # ---- load + keep what this rank owns
        # File sources: every rank parses 1/W of the bytes and one all-to-all-v per column moves the
        # rows to their owners (N10 + C4).  In-memory sources are identical on every rank -> filter.
        def load_owned(s, key):
            if s.data is not None and s.data.get("partitioned"):
                # in-memory source that already holds exactly this rank's rows (ids with |id| % world == rank, edges by
                # their source id) - e.g. generated or pre-sharded on the device: nothing to filter or move
                d = _load_source(s)
                if s.kind == "edge" and s.direction == REVERSED:
                    raise ValueError("partitioned in-memory edge sources must be directed (rows are owned by their source)")
                dst_own = d["b"][d["b"].abs() % W == r] if s.kind == "edge" else None
                return d, dst_own
            if s.data is None and W > 1 and cfg.sliced_load:
                d = _load_source(s, r, W)
                if s.kind == "edge" and s.direction == REVERSED:
                    d["a"], d["b"] = d["b"], d["a"]
                dst_own = None
                if s.kind == "edge":
                    ub = sorted_unique(d["b"])
                    dst_own = part.shuffle_rows({"a": ub}, ub.abs() % W, W, dev)["a"]
                return part.shuffle_rows(d, d[key].abs() % W, W, dev), dst_own
            d = _load_source(s)
            if s.kind == "edge" and s.direction == REVERSED:
                d["a"], d["b"] = d["b"], d["a"]
            dst_own = d["b"][d["b"].abs() % W == r] if s.kind == "edge" else None
            keep = (d[key].abs() % W == r).nonzero().flatten()
            return _take(d, keep), dst_own

        nd: Dict[str, List[Dict]] = {}
        for s in node_sources:
            d, _ = load_owned(s, "a")
            nd.setdefault(s.types, []).append(d)
        ed: Dict[str, List[Dict]] = {}
        ends: Dict[str, List[torch.Tensor]] = {}   # node type -> owned endpoint ids seen in edges
        for s in edge_sources:
            st, dt, et = s.types
            dk, own_dst = load_owned(s, "a")
            # endpoint id sets: edge files are usually grouped by src, so collapse runs before the real unique
            ends.setdefault(dt, []).append(torch.unique_consecutive(own_dst))
            ends.setdefault(st, []).append(torch.unique_consecutive(dk["a"]))
            ed.setdefault(et, []).append(dk)
            self.topology.add(et, st, dt)
        # ---- node tables
        types = sorted(set(list(nd.keys()) + list(ends.keys())))
        types = rt.all_gather_object(types)[0] if W > 1 else types
        for t in types:
            parts = nd.get(t, [])
            ids_src = torch.cat([p["a"].to(dev) for p in parts]) if parts else \
                torch.zeros(0, dtype=torch.int64, device=dev)
            ids_all = torch.cat([ids_src] + [e.to(dev) for e in ends.get(t, [])]) if (parts or t in ends) else ids_src
            idmap = IdMap.build(rt, ids_all)
            tab = NodeTable(rt, t, idmap)
            n = idmap.n_local
            dec = self.node_decoders.get(t, Decoder())
            rows = idmap._local_rows(ids_src.to(dev)) if ids_src.numel() else torch.zeros(0, dtype=torch.int64, device=dev)
            present = torch.zeros(n, dtype=torch.bool, device=dev)
            present[rows] = True
            tab.present = present
            merged = {k: (torch.cat([p[k].to(dev) for p in parts]) if parts and parts[0][k] is not None and k != "strs" else None)
                      for k in ("w", "label", "ts", "ia", "fa")}
            if dec.float_attr_num > 0:
                x = torch.full((n, dec.float_attr_num), float(cfg.default_float_attribute), device=dev)
                if merged["fa"] is not None:
                    x[rows] = merged["fa"].to(dev).float()
                tab.set_float(x, fdt)
            if dec.int_attr_num > 0:
                x = torch.full((n, dec.int_attr_num), int(cfg.default_int_attribute), dtype=torch.int64, device=dev)
                if merged["ia"] is not None:
                    x[rows] = merged["ia"].to(dev)
                tab.set_ints(x)
            if dec.labeled:
                x = torch.full((n,), int(cfg.default_label), dtype=torch.int64, device=dev)
                if merged["label"] is not None:
                    x[rows] = merged["label"].to(dev)
                tab.set_labels(x)
            if dec.weighted:
                x = torch.full((n,), float(cfg.default_weight), device=dev)
                if merged["w"] is not None:
                    x[rows] = merged["w"].to(dev).float()
                tab.set_weights(x)
            if dec.timestamped:
                x = torch.full((n,), int(cfg.default_timestamp), dtype=torch.int64, device=dev)
                if merged["ts"] is not None:
                    x[rows] = merged["ts"].to(dev)
                tab.set_timestamps(x)
            if dec.string_attr_num > 0:
                tab.str_dim = dec.string_attr_num
                arr = np.full((n, dec.string_attr_num), cfg.default_string_attribute, dtype=object)
                if parts and parts[0]["strs"] is not None:
                    arr[rows.cpu().numpy()] = np.concatenate([p["strs"] for p in parts])
                tab.strings = arr
            self.nodes[t] = tab
            for src_ in node_sources:          # g.node(..., option=gl.IndexOption()) -> KNN index on this table
                if src_.types == t and getattr(src_.option, "name", None) == "knn":
                    from ..ops import knn as _knn
                    _knn.build_index(tab, src_.option)
        # ---- edge shards
        for et in self.topology.edge_types():
            st, dt = self.topology.get_src_type(et), self.topology.get_dst_type(et)
            parts = ed.get(et, [])
            cat = lambda k: (torch.cat([p[k].to(dev) for p in parts]) if parts and parts[0][k] is not None else None)  # noqa: E731
            src = cat("a") if parts else torch.zeros(0, dtype=torch.int64, device=dev)
            dst = cat("b") if parts else torch.zeros(0, dtype=torch.int64, device=dev)
            src_tab, dst_tab = self.nodes[st], self.nodes[dt]
            src_rows = src_tab.idmap._local_rows(src)
            dst_vids = dst_tab.idmap.to_vid(dst)
            csr = CsrShard.from_coo(rt, et, st, dt, src_rows, dst_vids, src_tab.n_local, weights=cat("w"),
                                    ts=cat("ts"), labels=cat("label"), float_attrs=cat("fa"), int_attrs=cat("ia"))
            strs = [p["strs"] for p in parts if p["strs"] is not None]
            csr.strings = np.concatenate(strs)[csr._order.cpu().numpy()] if strs else None
            self.edges[et] = csr
            ip = csr.indptr.local
            src_tab.out_degrees[et] = ip[1:] - ip[:-1]
        # ---- statistics (GetCount / GetStats, graph_store.cc:278-317)
        for t, tab in self.nodes.items():
            self.stats[t] = rt.all_gather_object(int(tab.present.sum().item()) if tab.present is not None else tab.n_local)
        for et, csr in self.edges.items():
            self.stats[et] = rt.all_gather_object(csr.n_edges)
        rt.barrier()

    # ------------------------------------------------------------------ masked views (Graph.node_view)
    def add_node_view(self, base_type: str, masked_type: str, seed: int, nsplit: int, split_range):
        """Masked node table holding the ids of ``base_type`` with hash(id, seed) % nsplit in split_range.
        Every rank filters the ids it owns, so the view is partitioned like its base.  Collective."""
        base = self.nodes[base_type]
        rows = base.present.nonzero().flatten() if base.present is not None else \
            torch.arange(base.n_local, device=self.rt.device)
        vids = rows * self.rt.world + self.rt.rank
        ids = base.idmap.to_id(vids) if not base.idmap.dense else vids
        h = (ids ^ (int(seed) * 0x9E3779B97F4A7C15 & 0x7FFFFFFFFFFFFFFF)) & 0x7FFFFFFFFFFFFFFF
        h = ((h ^ (h >> 30)) * 0x5851F42D4C957F2D) & 0x7FFFFFFFFFFFFFFF      # splitmix-style mixing
        h = ((h ^ (h >> 27)) * 0x14057B7EF767814F) & 0x7FFFFFFFFFFFFFFF
        bucket = (h ^ (h >> 31)) % max(int(nsplit), 1)
        keep = ids[(bucket >= split_range[0]) & (bucket < split_range[1])]
        idmap = IdMap.build(self.rt, keep)
        tab = NodeTable(self.rt, masked_type, idmap)
        tab.present = torch.ones(idmap.n_local, dtype=torch.bool, device=self.rt.device)
        self.nodes[masked_type] = tab
        self.stats[masked_type] = self.rt.all_gather_object(idmap.n_local)
        return tab

    # ------------------------------------------------------------------ N17: hot-feature replica cache
    def build_feature_caches(self, capacity: int) -> Dict[str, int]:
        """Cache up to ``capacity`` remote feature rows per node type on every rank, hottest
        (largest global in-degree over all edge types pointing at the type) first.
        ``gl.set_local_node_cache_capacity(n)`` before ``g.init()`` calls this.  Collective."""
        rt = self.rt
        out: Dict[str, int] = {}
        if rt.world == 1 or capacity <= 0:
            return out
        for t, tab in self.nodes.items():
            if tab.feats is None:
                continue
            max_vid = max(int(n) for n in tab.nrows) * rt.world
            deg = torch.zeros(max_vid, dtype=torch.float32, device=rt.device)
            for et, csr in self.edges.items():
                if csr.dst_type != t or csr.indices is None:
                    continue
                idx = csr.indices.local
                idx = idx[(idx >= 0) & (idx < max_vid)]
                if idx.numel():
                    deg += torch.bincount(idx, minlength=max_vid).float()
            import torch.distributed as dist
            dist.all_reduce(deg)
            out[t] = tab.build_feature_cache(capacity, scores=deg)
        return out

    # ------------------------------------------------------------------ in-edges (lazy; collective)
    def reverse_csr(self, etype: str) -> CsrShard:
        """CSR of the in-edges of `etype`, partitioned by DESTINATION owner (for inV / in-degrees)."""
        if etype in self.reverse:
            return self.reverse[etype]
        from ..parallel import partition as part
        rt, W = self.rt, self.rt.world
        csr = self.edges[etype]
        st, dt = csr.src_type, csr.dst_type
        src_vids = csr._row_of_edge * W + rt.rank
        dst_vids = csr.indices.local
        w = csr.weights.local if csr.weights is not None else None
        ts = csr.ts.local if csr.ts is not None else None
        fwd = torch.arange(csr.n_edges, device=dst_vids.device)     # edge id = position in the forward CSR
        if W > 1:
            ok = dst_vids >= 0
            sorted_dst, order, counts = part.partition_by_owner(dst_vids[ok], W)
            sc = [int(x) for x in counts.tolist()]
            rc = part.exchange_counts(counts)
            dst_vids = part._all_to_all_v(sorted_dst, sc, rc)
            src_vids = part._all_to_all_v(src_vids[ok][order], sc, rc)
            fwd = part._all_to_all_v(fwd[ok][order], sc, rc)
            if w is not None:
                w = part._all_to_all_v(w[ok][order], sc, rc)
            if ts is not None:
                ts = part._all_to_all_v(ts[ok][order], sc, rc)
        else:
            ok = dst_vids >= 0
            dst_vids, src_vids, fwd = dst_vids[ok], src_vids[ok], fwd[ok]
            w = w[ok] if w is not None else None
            ts = ts[ok] if ts is not None else None
        rows = torch.div(dst_vids, W, rounding_mode="floor")
        # in-edge rows keep the forward edge's id, weight and timestamp: inE()/inV() then honour
        # topk / temporal filters and edge-attribute lookups address the ORIGINAL edge
        rev = CsrShard.from_coo(rt, etype + "#in", dt, st, rows, src_vids, self.nodes[dt].n_local, weights=w, ts=ts,
                                eids=fwd)
        self.reverse[etype] = rev
        ip = rev.indptr.local
        self.nodes[dt].in_degrees[etype] = ip[1:] - ip[:-1]
        return rev

    def ensure_indegree_weights(self, etype: str):
        """Per-edge weight = in-degree(dst) for InDegreeSampler (collective)."""
        from ..ops import gather as G
        csr = self.edges[etype]
        if csr.cumw_indeg is not None:
            return
        self.reverse_csr(etype)
        dt = self.nodes[csr.dst_type]
        indeg = self.rt.symm_from(dt.in_degrees[etype].to(torch.int64))
        vals = G.gather_any(self.rt, indeg, csr.indices.local, fill=0)
        csr.set_indegree_weights(vals)
