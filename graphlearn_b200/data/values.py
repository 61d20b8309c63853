"""Result objects of queries and samplers: ``Nodes``, ``Edges``, sparse variants,
``Layers`` / ``Layer`` and ``SubGraph``.

API parity with graphlearn/python/data/values.py (shapes and property names:
``ids [B] | [B,k]``, ``int_attrs/float_attrs/string_attrs [..., n]``,
``weights/labels/timestamps``, degrees dicts, ``offsets/indices/dense_shape``
for sparse objects, 1-based ``Layers.layer_nodes(i)``), but GPU-first inside:
every field is held as a **device tensor** (``.tensor(name)`` / ``.ids_t``) and
only converted to numpy when the numpy-style property is read, so a training
loop never bounces a batch through the host.  Attributes are looked up lazily
through ``graph.lookup_nodes`` exactly like the reference.
"""
from __future__ import annotations

from typing import Dict, Optional

import numpy as np
import torch


def _to_t(x, dtype=None):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x if dtype is None else x.to(dtype)
    a = np.asarray(x)
    if a.dtype.kind in ("U", "S", "O"):
        return a                          # strings stay on the host
    t = torch.from_numpy(np.ascontiguousarray(a))
    return t if dtype is None else t.to(dtype)


def _to_np(x):
    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    return np.asarray(x)


class Values(object):
    _FIELDS = ("int_attrs", "float_attrs", "string_attrs", "weights", "labels", "timestamps")

    def __init__(self, int_attrs=None, float_attrs=None, string_attrs=None, weights=None, labels=None,
                 timestamps=None, shape=None, graph=None):
        self._shape = shape
        self._graph = graph
        self._t: Dict[str, object] = {}
        self._inited = False
        for name, v in (("int_attrs", int_attrs), ("float_attrs", float_attrs), ("string_attrs", string_attrs),
                        ("weights", weights), ("labels", labels), ("timestamps", timestamps)):
            if v is not None:
                self._t[name] = _to_t(v)
                self._inited = True

    # ---- tensor (device) view
    def tensor(self, name) -> Optional[torch.Tensor]:
        """Device tensor of a field ('ids', 'float_attrs', 'labels', ...), reshaped to `shape`."""
        if name in self._FIELDS and name not in self._t:
            self._init()
        v = self._t.get(name)
        if v is None or not isinstance(v, torch.Tensor):
            return v
        return self._reshape_t(v, expand=name.endswith("_attrs"))

    def _reshape_t(self, v, expand=False):
        if v is None or self._shape is None or (hasattr(v, "numel") and v.numel() == 0):
            return v
        shp = tuple(self._shape)
        return v.reshape(shp + (-1,)) if expand else v.reshape(shp)

    def _np_field(self, name):
        if name not in self._t:
            self._init()
        v = self._t.get(name)
        if v is None:
            return None
        a = _to_np(v)
        if a.size == 0 or self._shape is None:
            return a
        shp = tuple(self._shape)
        return a.reshape(shp + (-1,)) if name.endswith("_attrs") else a.reshape(shp)

    int_attrs = property(lambda self: self._np_field("int_attrs"),
                         lambda self, v: self._t.__setitem__("int_attrs", _to_t(v)))
    float_attrs = property(lambda self: self._np_field("float_attrs"),
                           lambda self, v: self._t.__setitem__("float_attrs", _to_t(v)))
    string_attrs = property(lambda self: self._np_field("string_attrs"),
                            lambda self, v: self._t.__setitem__("string_attrs", _to_t(v)))
    weights = property(lambda self: self._np_field("weights"),
                       lambda self, v: self._t.__setitem__("weights", _to_t(v)))
    labels = property(lambda self: self._np_field("labels"),
                      lambda self, v: self._t.__setitem__("labels", _to_t(v)))
    timestamps = property(lambda self: self._np_field("timestamps"),
                          lambda self, v: self._t.__setitem__("timestamps", _to_t(v)))

    @property
    def shape(self):
        return self._shape

    @shape.setter
    def shape(self, shape):
        if not isinstance(shape, tuple):
            raise ValueError("shape must be a tuple, got {}.".format(type(shape)))
        self._shape = shape

    @property
    def graph(self):
        return self._graph

    @graph.setter
    def graph(self, g):
        self._graph = g

    def _init(self):
        if self._inited or self._graph is None:
            return
        self._inited = True
        try:
            if not self._get_decoder().has_property:
                return
        except AttributeError:
            return
        vals = self._lookup()
        for name in self._FIELDS:
            v = vals._t.get(name)
            if v is not None and name not in self._t:
                self._t[name] = v

    def _lookup(self):
        raise NotImplementedError

    def _get_decoder(self):
        raise NotImplementedError


class SparseBase(object):
    """Ragged results: ``offsets`` = per-row counts (reference naming), ``indices`` = (row, col) pairs."""

    def __init__(self, offsets, dense_shape):
        self._offsets = _to_np(offsets).astype(np.int64) if offsets is not None else None
        self._dense_shape = tuple(dense_shape) if dense_shape is not None else None
        self._indices = None
        self._it = 0
        self._cum = None

    @property
    def offsets(self):
        return self._offsets

    @offsets.setter
    def offsets(self, o):
        self._offsets = _to_np(o).astype(np.int64)
        self._indices = None

    @property
    def dense_shape(self):
        return self._dense_shape

    @dense_shape.setter
    def dense_shape(self, s):
        self._dense_shape = tuple(s)

    @property
    def indices(self):
        if self._indices is None:
            rows = np.repeat(np.arange(len(self._offsets)), self._offsets)
            cols = np.concatenate([np.arange(c) for c in self._offsets]) if len(self._offsets) else np.zeros(0, int)
            self._indices = np.stack([rows, cols.astype(np.int64)], 1) if rows.size else np.zeros((0, 2), np.int64)
        return self._indices

    def _bounds(self, i):
        if self._cum is None:
            self._cum = np.concatenate([[0], np.cumsum(self._offsets)])
        return int(self._cum[i]), int(self._cum[i + 1])

    def __iter__(self):
        self._it = 0
        return self

    def next(self):
        return self.__next__()


class Nodes(Values):
    def __init__(self, ids, node_type, int_attrs=None, float_attrs=None, string_attrs=None, weights=None,
                 labels=None, timestamps=None, shape=None, graph=None, vids=None):
        super().__init__(int_attrs, float_attrs, string_attrs, weights, labels, timestamps, shape, graph)
        t = _to_t(ids, torch.int64)
        if shape is None:
            self._shape = tuple(t.shape)
        else:
            n = int(np.prod(shape)) if len(shape) else 1
            if t.numel() == n:
                self._shape = tuple(shape)
            else:
                self._shape = tuple(t.shape) if len(shape) == 1 else (t.numel() // int(np.prod(shape[1:])),) + tuple(shape[-1:])
        self._t["ids"] = t.reshape(self._shape) if t.numel() else t
        if vids is not None:
            self._t["vids"] = _to_t(vids, torch.int64)
        self._type = node_type
        self._out_degrees = {}
        self._in_degrees = {}

    def _get_decoder(self):
        return self._graph.get_node_decoder(self._type)

    def _lookup(self):
        return self._graph.lookup_nodes(self._type, self._t["ids"], vids=self._t.get("vids"))

    @property
    def ids(self):
        return _to_np(self._t["ids"])

    @ids.setter
    def ids(self, ids):
        t = _to_t(ids, torch.int64)
        self._t["ids"] = t.reshape(self._shape) if self._shape and t.numel() else t

    @property
    def ids_t(self) -> torch.Tensor:
        return self._t["ids"]

    @property
    def vids_t(self) -> Optional[torch.Tensor]:
        """Internal virtual ids (row * world + owner) when known - lets kernels skip the id lookup."""
        return self._t.get("vids")

    @property
    def type(self):
        return self._type

    @type.setter
    def type(self, t):
        self._type = t

    @property
    def in_degrees(self):
        return self._in_degrees or None

    @property
    def out_degrees(self):
        return self._out_degrees or None

    def get_in_degrees(self, edge_type):
        if self._graph.get_topology().get_dst_type(edge_type) != self._type:
            raise ValueError("Nodes {} has no in edge with type {}".format(self._type, edge_type))
        if edge_type not in self._in_degrees:
            self._in_degrees[edge_type] = self._graph.in_degrees(self.ids, edge_type)
        return self._in_degrees[edge_type]

    def add_in_degrees(self, edge_type, degrees):
        self._in_degrees[edge_type] = _to_np(degrees)

    def get_out_degrees(self, edge_type):
        if self._graph.get_topology().get_src_type(edge_type) != self._type:
            raise ValueError("Nodes {} has no out edge with type {}".format(self._type, edge_type))
        if edge_type not in self._out_degrees:
            self._out_degrees[edge_type] = self._graph.out_degrees(self.ids, edge_type)
        return self._out_degrees[edge_type]

    def add_out_degrees(self, edge_type, degrees):
        self._out_degrees[edge_type] = _to_np(degrees)

    def embedding_agg(self, func="sum"):
        """[B, k] neighbours -> [B, float_attr_num] aggregated on the owning GPUs
        (Aggregator operators, graphlearn/python/data/values.py:346-379)."""
        if len(self.shape) != 2:
            raise ValueError("embedding_agg is for Nodes with 2 dimension, and the default aggregated dimension is axis=1")
        out = self._graph.aggregate_nodes(self._type, self._t["ids"].reshape(-1), func, k=self.shape[1],
                                          vids=self._t.get("vids"))
        return _to_np(out)


class SparseNodes(Nodes, SparseBase):
    def __init__(self, ids, offsets, dense_shape, node_type, int_attrs=None, float_attrs=None, string_attrs=None,
                 weights=None, labels=None, timestamps=None, graph=None, vids=None):
        t = _to_t(ids, torch.int64).reshape(-1)
        Nodes.__init__(self, t, node_type, int_attrs, float_attrs, string_attrs, weights, labels, timestamps,
                       shape=(int(t.numel()),), graph=graph, vids=vids)
        SparseBase.__init__(self, offsets, dense_shape)

    def __next__(self):
        if self._it >= len(self._offsets):
            raise StopIteration
        s, e = self._bounds(self._it)
        self._it += 1

        def cut(name):
            v = self._np_field(name) if (name in self._t or self._inited) else None
            return None if v is None else v[s:e]

        return Nodes(self.ids[s:e], self._type, cut("int_attrs"), cut("float_attrs"), cut("string_attrs"),
                     cut("weights"), cut("labels"), cut("timestamps"), graph=self._graph)

    def embedding_agg(self, func="sum"):
        offs = torch.from_numpy(np.concatenate([[0], np.cumsum(self._offsets)])).to(self._t["ids"].device)
        out = self._graph.aggregate_nodes(self._type, self._t["ids"].reshape(-1), func, offsets=offs,
                                          vids=self._t.get("vids"))
        return _to_np(out)


class Edges(Values):
    def __init__(self, src_ids=None, src_type=None, dst_ids=None, dst_type=None, edge_type=None, edge_ids=None,
                 src_nodes=None, dst_nodes=None, int_attrs=None, float_attrs=None, string_attrs=None, weights=None,
                 labels=None, timestamps=None, shape=None, graph=None, src_vids=None):
        super().__init__(int_attrs, float_attrs, string_attrs, weights, labels, timestamps, shape, graph)
        if src_nodes is not None and src_ids is None:
            src_ids, src_type = src_nodes.ids_t, src_nodes.type
        if dst_nodes is not None and dst_ids is None:
            dst_ids, dst_type = dst_nodes.ids_t, dst_nodes.type
        s = _to_t(src_ids, torch.int64)
        d = _to_t(dst_ids, torch.int64)
        base = d if d is not None else s
        if shape is None:
            self._shape = tuple(base.shape)
        else:
            self._shape = tuple(shape) if base.numel() == int(np.prod(shape)) else tuple(base.shape)
        if s is not None and d is not None and s.numel() != d.numel() and s.numel() > 0:
            s = s.reshape(-1, 1).expand(-1, d.numel() // s.numel())
        self._t["src_ids"] = s.reshape(self._shape) if s is not None and s.numel() else s
        self._t["dst_ids"] = d.reshape(self._shape) if d is not None and d.numel() else d
        e = _to_t(edge_ids, torch.int64)
        self._t["edge_ids"] = e.reshape(self._shape) if e is not None and e.numel() else e
        if src_vids is not None:
            self._t["src_vids"] = _to_t(src_vids, torch.int64)
        self._src_type, self._dst_type, self._edge_type = src_type, dst_type, edge_type
        self._src_nodes = src_nodes
        self._dst_nodes = dst_nodes

    def _get_decoder(self):
        return self._graph.get_edge_decoder(self._edge_type)

    def _lookup(self):
        if self._t.get("edge_ids") is None and self._t.get("dst_ids") is not None:
            # edges given by their end points only (g.get_edges(etype, src, dst)): resolve the ids first
            e = self._graph.find_edge_ids(self._edge_type, self._t["src_ids"], self._t["dst_ids"])
            self._t["edge_ids"] = e.reshape(self._shape)
        return self._graph.lookup_edges(self._edge_type, self._t["src_ids"], self._t["edge_ids"],
                                        src_vids=self._t.get("src_vids"))

    src_ids = property(lambda self: _to_np(self._t.get("src_ids")))
    dst_ids = property(lambda self: _to_np(self._t.get("dst_ids")))
    edge_ids = property(lambda self: _to_np(self._t.get("edge_ids")))
    src_type = property(lambda self: self._src_type)
    dst_type = property(lambda self: self._dst_type)
    edge_type = property(lambda self: self._edge_type)
    type = property(lambda self: (self._src_type, self._dst_type, self._edge_type))

    @property
    def src_nodes(self):
        if self._src_nodes is None and self._t.get("src_ids") is not None:
            self._src_nodes = Nodes(self._t["src_ids"], self._src_type, shape=self._shape, graph=self._graph)
        return self._src_nodes

    @src_nodes.setter
    def src_nodes(self, n):
        self._src_nodes = n

    @property
    def dst_nodes(self):
        if self._dst_nodes is None and self._t.get("dst_ids") is not None:
            self._dst_nodes = Nodes(self._t["dst_ids"], self._dst_type, shape=self._shape, graph=self._graph)
        return self._dst_nodes

    @dst_nodes.setter
    def dst_nodes(self, n):
        self._dst_nodes = n


class SparseEdges(Edges, SparseBase):
    def __init__(self, src_ids, src_type, dst_ids, dst_type, edge_type, offsets, dense_shape, edge_ids=None,
                 int_attrs=None, float_attrs=None, string_attrs=None, weights=None, labels=None, timestamps=None,
                 graph=None):
        d = _to_t(dst_ids, torch.int64).reshape(-1)
        s = _to_t(src_ids, torch.int64).reshape(-1)
        Edges.__init__(self, s, src_type, d, dst_type, edge_type, edge_ids, None, None, int_attrs, float_attrs,
                       string_attrs, weights, labels, timestamps, shape=(int(d.numel()),), graph=graph)
        SparseBase.__init__(self, offsets, dense_shape)

    def __next__(self):
        if self._it >= len(self._offsets):
            raise StopIteration
        s, e = self._bounds(self._it)
        self._it += 1
        eid = self.edge_ids
        return Edges(self.src_ids[s:e], self._src_type, self.dst_ids[s:e], self._dst_type, self._edge_type,
                     None if eid is None else eid[s:e], graph=self._graph)


class Layer(object):
    def __init__(self, nodes, edges=None, shape=None):
        self._nodes, self._edges, self._shape = nodes, edges, shape

    nodes = property(lambda self: self._nodes, lambda self, v: setattr(self, "_nodes", v))
    edges = property(lambda self: self._edges, lambda self, v: setattr(self, "_edges", v))
    shape = property(lambda self: self._shape, lambda self, v: setattr(self, "_shape", v))


class Layers(object):
    """Multi-hop sampling result; layer ids are 1-based like the reference."""

    def __init__(self, layers=None):
        self.layers = list(layers) if layers else []

    def _check(self, layer_id):
        layer_id -= 1
        if not isinstance(self.layers, list) or layer_id < 0 or layer_id >= len(self.layers):
            raise ValueError("layer id beyond the layers length.")
        return layer_id

    def layer(self, layer_id):
        return self.layers[self._check(layer_id)]

    def layer_size(self, layer_id):
        return self.layers[self._check(layer_id)].shape

    def layer_nodes(self, layer_id):
        return self.layers[self._check(layer_id)].nodes

    def layer_edges(self, layer_id):
        return self.layers[self._check(layer_id)].edges

    def set_layer_nodes(self, layer_id, nodes):
        self.layers[self._check(layer_id)].nodes = nodes

    def set_layer_edges(self, layer_id, edges):
        self.layers[self._check(layer_id)].edges = edges

    def append_layer(self, layer):
        self.layers.append(layer)


class SubGraph(object):
    """Induced subgraph: ``edge_index [2, m]`` indexes into ``nodes``."""

    def __init__(self, edge_index, nodes, edges=None, **kwargs):
        self._edge_index = _to_t(edge_index, torch.int64)
        self._nodes = nodes
        self._edges = edges
        for k, v in kwargs.items():
            setattr(self, k, v)

    @property
    def edge_index(self):
        return _to_np(self._edge_index)

    @property
    def edge_index_t(self):
        return self._edge_index

    nodes = property(lambda self: self._nodes)
    edges = property(lambda self: self._edges)

    @property
    def num_nodes(self):
        return int(self._nodes.ids_t.numel())

    @property
    def num_edges(self):
        return int(self._edge_index.size(1))

    @property
    def keys(self):
        """names of the attributes that are set: edge_index, nodes, edges and any extras such as dist_to_src / dist_to_dst
        (nn/subgraph.py ``keys``)"""
        base = ["edge_index", "nodes"] + (["edges"] if self._edges is not None else [])
        return base + [k for k, v in self.__dict__.items() if not k.startswith("_") and v is not None]
