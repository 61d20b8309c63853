"""PyTorch model layer (``gl.nn``): the math of graphlearn/python/nn/tf/* re-implemented as
torch Modules, with the GraphSAGE layer on the fused sm_90a kernel."""
from . import loss  # noqa: F401
from torch.nn import Module  # noqa: F401  (nn/tf/module.py: the base class of every layer / model)

from .conv import (EgoConv, EgoGATConv, EgoGINConv, EgoLayer, EgoRGCNConv, EgoSAGEConv, EgoTGATConv,  # noqa: F401
                   LinearLayer, SubConv, TimeEncoder)
from .norm import compute_norm, compute_saint_norm  # noqa: F401
from .data import BatchGraph, Data, EgoGraph, HeteroBatchGraph, TemporalGraph  # noqa: F401
from .dataset import (Batch, Collater, Dataset, PyGDataLoader, SubGraphData, TemporalData, TemporalDataLoader,  # noqa: F401
                      TemporalDataset, TorchDataset, worker_init_fn)
from .embedding import ShardedEmbedding  # noqa: F401
from .feature import DynamicEmbedding, FeatureEncoder  # noqa: F401
from .feature_column import (DynamicEmbeddingColumn, DynamicSparseEmbeddingColumn, EmbeddingColumn, FeatureColumn,  # noqa: F401
                             FeatureGroup, FeatureHandler, FusedEmbeddingColumn, NumericColumn, PartitionableColumn,
                             SparseEmbeddingColumn)
from .hetero import (BipartiteSAGEConv, HeteroConv, HeteroSubGraph, LinkPredictor, SubGraphInducer,  # noqa: F401
                     SubGraphProcessor)
from .sparse_conv import GATConv, GCNConv, SAGEConv, segment_softmax  # noqa: F401
from .sparse_conv import segment_softmax as unsorted_segment_softmax  # noqa: F401  (nn/tf/utils/softmax.py name)
from .utils import Config, conf  # noqa: F401  (nn/tf/config.py)
from .utils import (SyncBarrierHook, bootstrap, get_cluster_spec, get_counts, get_num_client, get_rank, get_world_size,  # noqa: F401
                    is_server_launched, launch_server, set_client_num)
