"""Typed, process-global configuration (N1 of SURVEY.md).

Mirrors every ``gl.set_*`` of the reference (graphlearn/python/config.py:23-128,
defaults from graphlearn/src/common/base/config.cc:77-119) on top of one
dataclass instead of ~40 C++ globals.  Flags that only made sense for the gRPC /
thread-pool runtime are kept as inert fields so user scripts keep working.
"""
from __future__ import annotations

import dataclasses
import os

PADDING_REPLICATE = 0
PADDING_CIRCULAR = 1
REPLICATE = PADDING_REPLICATE
CIRCULAR = PADDING_CIRCULAR

TRACKER_RPC = 0
TRACKER_FS = 1


@dataclasses.dataclass
class Config:
    # --- semantics that matter on the GPU engine
    default_neighbor_id: int = 0
    default_int_attribute: int = 0
    default_float_attribute: float = 0.0
    default_string_attribute: str = ""
    default_weight: float = 0.0
    default_label: int = -1
    default_timestamp: int = -1
    padding_mode: int = PADDING_CIRCULAR
    sampling_retry_times: int = 5
    default_full_nbr_num: int = 100
    neg_sampling_retry_times: int = 5
    ignore_invalid: bool = False
    shuffle_buffer_size: int = 10240
    data_init_batch_size: int = 10240
    dataset_capacity: int = 10
    tape_capacity: int = 10
    storage_mode: int = 2
    local_node_cache_capacity: int = 0
    actor_local_shard_count: int = 1
    sliced_load: bool = True          # each rank parses 1/world of a file, rows are shuffled to owners
    knn_metric: int = 0          # 0 = L2, 1 = inner product
    field_delimiter: str = "\t"
    vineyard_graph_id: int = 0
    vineyard_ipc_socket: str = ""
    # --- runtime knobs
    timeout: int = 60
    retry_times: int = 10
    inter_threadnum: int = 32
    intra_threadnum: int = 32
    inmemory_queuesize: int = 10240
    rpc_message_max_size: int = 16 * 1024 * 1024
    tracker_mode: int = TRACKER_FS
    tracker: str = "/tmp/graphlearn/"
    deploy_mode: int = 0
    client_id: int = 0
    client_count: int = 1
    server_id: int = 0
    server_count: int = 1
    server_hosts: str = ""
    # --- GPU engine specific
    feature_dtype: str = "fp32"          # fp32 | bf16 | fp8 (e4m3, bf16 scale per 32 elements)   storage of float tables in HBM
    loader_threads: int = 0           # 0 = auto: all cores divided by the number of ranks on the box
    use_peer_kernels: bool = True        # False -> torch.distributed (NCCL/gloo) baseline path
    dedup_feature_pull: bool = False     # attribute lookups of GSL results fetch every distinct row once (ops/gather.py)
    native_csr_build: bool = True        # CUDA shards: counting build (csrc/csr_build.cu) instead of two global stable sorts
    feature_row_align: int = 128         # bytes: feature rows wider than half of this start on such a boundary (16 = dense rows)
    seed: int = 0
    actor_enabled: bool = False


def _from_env(cfg: "Config") -> "Config":
    """GLB_<FIELD> environment variables override the int / bool / float / str defaults (e.g. GLB_FEATURE_ROW_ALIGN=16)"""
    import os
    for f in dataclasses.fields(cfg):
        v = os.environ.get("GLB_" + f.name.upper())
        if v is None:
            continue
        cur = getattr(cfg, f.name)
        if isinstance(cur, bool):
            setattr(cfg, f.name, v.lower() not in ("0", "false", "no", ""))
        elif isinstance(cur, (int, float, str)):
            setattr(cfg, f.name, type(cur)(v))
    return cfg


_CFG = _from_env(Config())


def get() -> Config:
    return _CFG


def reset():
    global _CFG
    _CFG = _from_env(Config())
    return _CFG


def _setter(field, cast=lambda x: x):
    def f(value):
        setattr(_CFG, field, cast(value))
    f.__name__ = "set_" + field
    f.__doc__ = "Set global flag `%s` (reference: graphlearn/python/config.py)." % field
    return f


set_default_neighbor_id = _setter("default_neighbor_id", int)
set_default_int_attribute = _setter("default_int_attribute", int)
set_default_float_attribute = _setter("default_float_attribute", float)
set_default_string_attribute = _setter("default_string_attribute", str)
set_default_weight = _setter("default_weight", float)
set_default_label = _setter("default_label", int)
set_default_timestamp = _setter("default_timestamp", int)
set_sampling_retry_times = _setter("sampling_retry_times", int)
set_default_full_nbr_num = _setter("default_full_nbr_num", int)
set_neg_sampling_retry_times = _setter("neg_sampling_retry_times", int)
set_ignore_invalid = _setter("ignore_invalid", bool)
set_shuffle_buffer_size = _setter("shuffle_buffer_size", int)
set_data_init_batch_size = _setter("data_init_batch_size", int)
set_dataset_capacity = _setter("dataset_capacity", int)
set_tape_capacity = _setter("tape_capacity", int)
set_storage_mode = _setter("storage_mode", int)
set_local_node_cache_capacity = _setter("local_node_cache_capacity", int)
set_knn_metric = _setter("knn_metric", int)
set_field_delimiter = _setter("field_delimiter", str)
set_timeout = _setter("timeout", int)
set_retry_times = _setter("retry_times", int)
set_inter_threadnum = _setter("inter_threadnum", int)
set_intra_threadnum = _setter("intra_threadnum", int)
set_inmemory_queuesize = _setter("inmemory_queuesize", int)
set_rpc_message_max_size = _setter("rpc_message_max_size", int)
set_tracker_mode = _setter("tracker_mode", int)
set_tracker = _setter("tracker", str)
set_deploy_mode = _setter("deploy_mode", int)
set_client_id = _setter("client_id", int)
set_client_count = _setter("client_count", int)
set_server_id = _setter("server_id", int)
set_server_count = _setter("server_count", int)
set_server_hosts = _setter("server_hosts", str)
set_vineyard_graph_id = _setter("vineyard_graph_id", int)
set_vineyard_ipc_socket = _setter("vineyard_ipc_socket", str)
set_feature_dtype = _setter("feature_dtype", str)
set_loader_threads = _setter("loader_threads", int)
set_use_peer_kernels = _setter("use_peer_kernels", bool)
set_feature_row_align = _setter("feature_row_align", int)
set_native_csr_build = _setter("native_csr_build", bool)
set_dedup_feature_pull = _setter("dedup_feature_pull", bool)
set_seed = _setter("seed", int)


# exact reference spellings (graphlearn/python/config.py:77,114,118)
set_datainit_batchsize = set_data_init_batch_size
set_sampler_retry_times = set_sampling_retry_times


def set_actor_local_shard_count(count):
    """Actor engine knob (per-core shards of the hiactor runtime); accepted for script parity - the SM grid is
    the sharded executor here, there is nothing to size."""
    assert isinstance(count, int) and count > 0
    _CFG.actor_local_shard_count = int(count)


def set_inner_threadnum(n):
    """Reference quirk kept for parity: `set_inner_threadnum` sets the INTER pool
    (graphlearn/python/c/py_export.cc:51)."""
    _CFG.inter_threadnum = int(n)


def set_padding_mode(mode):
    assert mode in (PADDING_REPLICATE, PADDING_CIRCULAR)
    _CFG.padding_mode = int(mode)


def set_default_attribute(int_value=None, float_value=None, string_value=None):
    if int_value is not None:
        _CFG.default_int_attribute = int(int_value)
    if float_value is not None:
        _CFG.default_float_attribute = float(float_value)
    if string_value is not None:
        _CFG.default_string_attribute = str(string_value)


def enable_actor():
    """The reference switches to its hiactor runtime (graphlearn/src/service/server.cc:52-60): per-core sharded stores
    + (data-size aware) tape dispatch.  On the GPU the SM grid is the sharded executor; what the flag turns on is the
    balanced batch dispatch of engine/dispatch.py: multi-rank GSL root traversals pool their seed batches every epoch
    and hand every rank the same number of batches with balanced first-hop work."""
    _CFG.actor_enabled = True
