"""graphlearn_b200 - an H100-native distributed GNN training engine with the
capabilities and user API of alibaba/graph-learn (``import graphlearn_b200 as gl``).

Public surface mirrors graphlearn/__init__.py:16-40: ``gl.Graph``, ``gl.Dataset``,
``gl.Decoder``, ``gl.Mask``, ``gl.NODE / EDGE_SRC / EDGE_DST``, padding modes,
``gl.KnnOption``, errors and every ``gl.set_*`` flag; ``gl.nn`` holds the
PyTorch model layer.
"""
from __future__ import annotations

from . import config as _config
from .config import *  # noqa: F401,F403  (all set_* functions + constants)
from .config import CIRCULAR, REPLICATE, enable_actor  # noqa: F401
from .data.decoder import Decoder  # noqa: F401
from .data.feature_spec import FeatureSpec  # noqa: F401
from .data.values import Edges, Layer, Layers, Nodes, SparseEdges, SparseNodes, SubGraph, Values  # noqa: F401
from .errors import *  # noqa: F401,F403
from .errors import OutOfRangeError  # noqa: F401
from .graph import EDGE_DST, EDGE_SRC, NODE, Graph  # noqa: F401
from .gsl.dataset import Dataset  # noqa: F401
from .data.feature_spec import (DenseSpec, DynamicMultivalSpec, DynamicSparseSpec, MultivalSpec,  # noqa: F401
                                SparseSpec)
from .errors import BaseError  # noqa: F401
from .ops.knn import KnnOperator, KnnOption  # noqa: F401
from .sampler.negative_sampler import (ConditionalNegativeSampler, InDegreeNegativeSampler,  # noqa: F401
                                       NegativeSampler, NodeWeightNegativeSampler, RandomNegativeSampler)
from .sampler.neighbor_sampler import (EdgeWeightNeighborSampler, FullNeighborSampler,  # noqa: F401
                                       InDegreeNeighborSampler, NeighborSampler, RandomNeighborSampler,
                                       RandomWithoutReplacementNeighborSampler, TopkNeighborSampler)
from .sampler.edge_sampler import ByOrderEdgeSampler, EdgeSampler, RandomEdgeSampler, ShuffleEdgeSampler  # noqa: F401
from .sampler.node_sampler import ByOrderNodeSampler, NodeSampler, RandomNodeSampler, ShuffleNodeSampler  # noqa: F401
from .sampler.subgraph_sampler import SubGraphSampler  # noqa: F401
from .ops.sampling import LocalAdjacency, register_sampler, registered_samplers, unregister_sampler  # noqa: F401
from .utils import deprecated  # noqa: F401
from . import io  # noqa: F401  (gl.io.register_file_system, read_table, save_embeddings)
from .store.graph_store import Topology  # noqa: F401
from .utils import Mask, get_mask_type, strategy2op  # noqa: F401

__version__ = "0.1.0"

from . import nn  # noqa: E402,F401  (gl.nn, like the reference's `import graphlearn.python.nn as nn`)


class IndexOption(object):
    """KNN index options of the reference (graphlearn/python/c/py_export.cc): ``index_type`` in
    flat | ivfflat | ivfpq (+ the ``gpu_`` variants); flat = fused wgmma scan, ivfflat = k-means lists scanned
    exactly, ivfpq = the same lists with ``m`` one-byte product-quantiser codes per row, scored by look-up tables and
    re-ranked exactly (ops/knn.py)."""

    def __init__(self):
        self.name = "knn"
        self.index_type = "flat"
        self.nlist = 0
        self.nprobe = 0
        self.m = 0


def get_cluster(*args, **kwargs):
    from .cluster import get_cluster as _gc
    return _gc(*args, **kwargs)


def get_config():
    return _config.get()
