"""Rank bootstrap + symmetric (peer-mapped) memory registry.

Replaces the reference's cluster bring-up: gRPC services, FS/RPC coordinators,
naming engine and channel manager (graphlearn/src/service/dist/*.cc, SURVEY
R14-R18).  One process per GPU; ``torch.distributed`` (NCCL on GPU, gloo on
CPU) is used ONLY for rendezvous, IPC-handle exchange and as the baseline
collective path.  Afterwards every rank holds a peer-pointer table for every
sharded array and the sm_90a kernels dereference peer HBM directly.
"""
from __future__ import annotations

import os
from typing import List, Optional, Sequence

import torch
import torch.distributed as dist

from .. import _build

MAX_WORLD = 8
_DTYPE_CODE = {torch.float32: 0, torch.bfloat16: 1, torch.int64: 2, torch.int32: 3, torch.uint8: 4}


def native():
    """The compiled extension (raises loudly when it is missing)."""
    global _NATIVE
    if _NATIVE is None:
        _NATIVE = _build.load()
    return _NATIVE


_NATIVE = None


class SymmTensor:
    """A tensor allocated identically on every rank whose peers are mapped
    into this process (CUDA IPC).  ``local`` is this rank's shard; ``ptrs[r]``
    is the address of rank r's shard as seen from THIS process."""

    def __init__(self, local: torch.Tensor, ptrs: List[int], nrows: List[int], owned_ptr: int = 0,
                 peer_mapped: Optional[List[int]] = None):
        self.local = local
        self.ptrs = ptrs
        self.nrows = nrows
        self._owned_ptr = owned_ptr
        self._peer_mapped = peer_mapped or []

    @property
    def world(self):
        return len(self.ptrs)


class Runtime:
    _inst: Optional["Runtime"] = None

    def __init__(self):
        self.rank = 0
        self.world = 1
        self.local_rank = 0
        self.device = torch.device("cpu")
        self.initialized = False
        self.owns_pg = False
        self._symm: List[SymmTensor] = []

    # ------------------------------------------------------------------ bootstrap
    @classmethod
    def get(cls) -> "Runtime":
        if cls._inst is None:
            cls._inst = Runtime()
        return cls._inst

    def init(self, device: Optional[str] = None, backend: Optional[str] = None) -> "Runtime":
        if self.initialized:
            return self
        env_world = int(os.environ.get("WORLD_SIZE", "1"))
        use_cuda = torch.cuda.is_available() and device != "cpu"
        if dist.is_available() and dist.is_initialized():
            self.rank, self.world = dist.get_rank(), dist.get_world_size()
        elif env_world > 1:
            os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
            os.environ.setdefault("MASTER_PORT", "29533")
            self.local_rank = int(os.environ.get("LOCAL_RANK", os.environ.get("RANK", "0")))
            if use_cuda:
                torch.cuda.set_device(self.local_rank)
            dist.init_process_group(backend or ("nccl" if use_cuda else "gloo"),
                                    device_id=torch.device("cuda", self.local_rank) if use_cuda else None)
            self.owns_pg = True
            self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.local_rank = int(os.environ.get("LOCAL_RANK", str(self.rank)))
        if use_cuda:
            torch.cuda.set_device(self.local_rank)
            self.device = torch.device("cuda", self.local_rank)
        else:
            self.device = torch.device("cpu")
        if self.world > MAX_WORLD:
            raise RuntimeError("single-box engine: world size must be <= %d" % MAX_WORLD)
        self.initialized = True
        return self

    def shutdown(self):
        self.free_all()
        if self.owns_pg and dist.is_initialized():
            dist.destroy_process_group()
        self.initialized = False
        Runtime._inst = None

    @property
    def is_cuda(self):
        return self.device.type == "cuda"

    def barrier(self):
        if self.world > 1:
            if self.is_cuda:
                torch.cuda.synchronize()
            dist.barrier()

    def all_gather_object(self, obj):
        if self.world == 1:
            return [obj]
        out = [None] * self.world
        dist.all_gather_object(out, obj)
        return out

    # ------------------------------------------------------------------ symmetric memory
    def symm_from(self, t: torch.Tensor) -> SymmTensor:
        """Copy `t` into freshly allocated symmetric memory and map all peers."""
        st = self.symm_empty(tuple(t.shape), t.dtype)
        st.local.copy_(t)
        if self.is_cuda:
            torch.cuda.synchronize()
        self.barrier()
        return st

    def symm_empty(self, shape: Sequence[int], dtype: torch.dtype) -> SymmTensor:
        """Collective: every rank allocates its shard (shapes may differ in dim 0)."""
        shape = tuple(int(s) for s in shape)
        nrows_local = shape[0] if len(shape) > 0 else 1
        if not self.is_cuda:
            local = torch.zeros(shape, dtype=dtype)
            nrows = self.all_gather_object(nrows_local)
            ptrs = [0] * self.world
            ptrs[self.rank] = local.data_ptr()
            st = SymmTensor(local, ptrs, nrows)
            self._symm.append(st)
            return st
        C = native()
        numel = 1
        for s in shape:
            numel *= s
        nbytes = max(numel, 1) * torch.empty((), dtype=dtype).element_size()
        dev = self.device.index
        ptr = C.symm_alloc(nbytes, dev)
        local = C.tensor_from_ptr(ptr, list(shape), _DTYPE_CODE[dtype], dev)
        if self.world == 1:
            st = SymmTensor(local, [ptr], [nrows_local], owned_ptr=ptr)
            self._symm.append(st)
            return st
        handle = C.ipc_get_handle(ptr, dev)
        gathered = self.all_gather_object((handle, nrows_local))
        ptrs, nrows, mapped = [], [], []
        for r, (h, n) in enumerate(gathered):
            nrows.append(n)
            if r == self.rank:
                ptrs.append(ptr)
            else:
                p = C.ipc_open_handle(h, dev)
                ptrs.append(p)
                mapped.append(p)
        st = SymmTensor(local, ptrs, nrows, owned_ptr=ptr, peer_mapped=mapped)
        self._symm.append(st)
        return st

    def free_all(self):
        if self.is_cuda and self._symm:
            C = native()
            torch.cuda.synchronize()
            self.barrier()
            dev = self.device.index
            for st in self._symm:
                for p in st._peer_mapped:
                    try:
                        C.ipc_close_handle(p, dev)
                    except Exception:
                        pass
            self.barrier()
            for st in self._symm:
                if st._owned_ptr:
                    try:
                        C.symm_free(st._owned_ptr, dev)
                    except Exception:
                        pass
        self._symm = []


def runtime() -> Runtime:
    return Runtime.get()


def init(device: Optional[str] = None, backend: Optional[str] = None) -> Runtime:
    return Runtime.get().init(device=device, backend=backend)


def bootstrap_cluster(task_index: int, task_count: int, tracker: Optional[str] = None, hosts: Optional[str] = None,
                      device: Optional[str] = None, timeout_s: float = 600.0) -> None:
    """Form the process group WITHOUT torchrun, the way the reference's worker mode is launched: N independent processes call
    ``g.init(task_index=i, task_count=N, tracker=<shared dir>)`` (file-system tracker, graph.py:445-464 /
    fs_coordinator.cc) or ``g.init(..., hosts="ip:port,ip:port")`` (RPC tracker with an explicit host list).  The tracker
    directory becomes a ``torch.distributed`` file-store rendezvous, the first host a TCP rendezvous; like the reference, a
    tracker directory must be fresh for every job."""
    if dist.is_available() and dist.is_initialized():
        return
    import datetime
    use_cuda = torch.cuda.is_available() and device != "cpu"
    os.environ["RANK"], os.environ["WORLD_SIZE"] = str(int(task_index)), str(int(task_count))
    os.environ.setdefault("LOCAL_RANK", str(int(task_index)))
    if hosts:
        first = hosts.split(",")[0].strip()
        method = "tcp://" + first
    else:
        d = os.path.abspath(tracker or "/tmp/graphlearn")
        os.makedirs(d, exist_ok=True)
        path = os.path.join(d, "glb_rendezvous_%d" % int(task_count))
        # a file store removes its file when the job ends cleanly; one left behind by a CRASHED job would poison this one:
        # task 0 deletes a rendezvous file that is older than two minutes, the others wait until it is gone or fresh
        import time as _time
        stale = lambda: os.path.exists(path) and _time.time() - os.path.getmtime(path) > 120     # noqa: E731
        if int(task_index) == 0:
            if stale():
                try:
                    os.remove(path)
                except OSError:
                    pass
        else:
            t0 = _time.time()
            while stale() and _time.time() - t0 < timeout_s:
                _time.sleep(0.2)
        method = "file://" + path
    if use_cuda:
        torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl" if use_cuda else "gloo", init_method=method, rank=int(task_index), world_size=int(task_count),
                            timeout=datetime.timedelta(seconds=timeout_s))
    Runtime.get().owns_pg = True


# ---------------------------------------------------------------------- descriptors
def _pad8(xs, fill=0):
    xs = list(xs)
    return xs + [fill] * (MAX_WORLD - len(xs))


def make_csr_desc(world, nrows, indptr, indices, eids=None, cumw=None, ts=None, sorted_idx=None) -> torch.Tensor:
    """CPU int64[49] descriptor consumed by the sampling kernels (see csrc/sampling.cu); 57 entries when the id-sorted
    copy of the rows (``sorted_idx``, node2vec membership tests) is present."""
    z = [0] * world
    vals = [world] + _pad8(nrows) + _pad8(indptr) + _pad8(indices) + _pad8(eids or z) + \
        _pad8(cumw or z) + _pad8(ts or z)
    if sorted_idx is not None:
        vals += _pad8(sorted_idx)
    return torch.tensor(vals, dtype=torch.int64)


def make_table_desc(world, dim, stride, dtype, nrows, ptrs, cache=None) -> torch.Tensor:
    """CPU int64[20] descriptor of a row-sharded dense table (see csrc/host_utils.h);
    ``cache=(rank, cache_map_ptr, cache_rows_ptr)`` appends the replica-cache triple (23 entries)."""
    # 2 = fp8 e4m3 block-scaled rows (byte table; `stride` counts bytes, see csrc/host_utils.h)
    code = 0 if dtype == torch.float32 else 2 if dtype in (torch.float8_e4m3fn, torch.uint8) else 1
    vals = [world, dim, stride, code] + _pad8(nrows) + _pad8(ptrs)
    if cache is not None:
        vals += [int(cache[0]), int(cache[1]), int(cache[2])]
    return torch.tensor(vals, dtype=torch.int64)


def local_table_desc(t: torch.Tensor) -> torch.Tensor:
    """Descriptor of a plain local [n, d] tensor (world = 1, vid == row)."""
    assert t.dim() == 2 and t.stride(1) == 1
    assert t.dtype in (torch.float32, torch.bfloat16)
    return make_table_desc(1, t.size(1), t.stride(0), t.dtype, [t.size(0)], [t.data_ptr()])
