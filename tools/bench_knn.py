"""KNN search throughput (K10): flat scan (wgmma score GEMM + fused top-k) and IVF-flat on N x d database vectors, recall@k
against an fp32 brute-force oracle.  1 GPU: `python tools/bench_knn.py`; N GPUs: torchrun (database sharded by id % world,
peer-memory k-way merge)."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from graphlearn_b200.ops import knn as K  # noqa: E402
from graphlearn_b200.parallel.runtime import init  # noqa: E402
from graphlearn_b200.store.shards import IdMap, NodeTable  # noqa: E402

rt = init()
dev, W = rt.device, rt.world
N, d, k = int(os.environ.get("KNN_N", 2_000_000)), 128, 10
n_local = (N - rt.rank + W - 1) // W
g = torch.Generator(device=dev).manual_seed(1 + rt.rank)
centers = torch.randn(256, d, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
x = centers[torch.randint(0, 256, (n_local,), device=dev, generator=g)] + 0.3 * torch.randn(n_local, d, device=dev, generator=g)
tab = NodeTable(rt, "v", IdMap(rt, torch.arange(n_local, device=dev) * W + rt.rank, dense=True))
tab.set_float(x, torch.bfloat16)
gq = torch.Generator(device=dev).manual_seed(99)
res = {"what": "KNN search on %d x %d bf16 vectors over %d GPU(s), k = %d, L2" % (N, d, W, k), "n_gpus": W}


def timed(fn, reps=5):
    fn(); torch.cuda.synchronize(); rt.barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record(); torch.cuda.synchronize(); rt.barrier()
    return e0.elapsed_time(e1) / reps


for B in (64, 1024):
    q = centers[torch.randint(0, 256, (B,), device=dev, generator=gq)] + 0.3 * torch.randn(B, d, device=dev, generator=gq)
    tab._knn_option = ("flat", 0, 0)
    ms = timed(lambda: K.search(rt, tab, q, k, 0))
    ids, dist_ = K.search(rt, tab, q, k, 0)
    res["flat_B%d" % B] = {"ms_per_batch": round(ms, 3), "qps": round(B / ms * 1e3), "scanned_GB_per_s": round(N * d * 2 / (ms * 1e-3) / 1e9, 1)}
    if W == 1 and B == 64:        # recall vs fp32 brute force on the bf16-rounded database
        xf = tab.feats.local[:, :d].float()
        ref = torch.cdist(q, xf).topk(k, largest=False).indices
        hit = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ids.cpu(), ref.cpu()))
        res["flat_recall_at_%d" % k] = hit / (B * k)
    tab._knn_option = ("ivfflat", 1024, 16)
    tab._knn_index = None
    K.search(rt, tab, q, k, 0)    # builds the index (k-means) once
    ms = timed(lambda: K.search(rt, tab, q, k, 0))
    ids2, _ = K.search(rt, tab, q, k, 0)
    rec = sum(len(set(a.tolist()) & set(b.tolist())) for a, b in zip(ids2.cpu(), ids.cpu())) / (B * k)
    res["ivfflat_nlist1024_nprobe16_B%d" % B] = {"ms_per_batch": round(ms, 3), "qps": round(B / ms * 1e3), "recall_vs_flat": round(rec, 4)}
if rt.rank == 0:
    print(json.dumps(res))
rt.shutdown()
