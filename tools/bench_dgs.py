"""DGS benchmark against the reference's published numbers (docs/en/dgs/intro.md:25-29: 2-hop query P99 <= 20 ms,
20,000 QPS, 110 MB/s update ingest on a 64-core node): streaming ingest throughput, 2-hop query latency and QPS of
the HBM-resident sampler service on one H100."""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from graphlearn_b200.dgs import DynamicGraphService, QueryPlan

dev = "cuda" if torch.cuda.is_available() else "cpu"
NU, NI, FD = 1_000_000, 1_000_000, 32
schema = {"vertices": {"u": {"count": NU, "feat_dim": FD}, "i": {"count": NI, "feat_dim": FD}},
          "edges": {"click": {"src": "u", "dst": "i"}, "sim": {"src": "i", "dst": "i"}}}
svc = DynamicGraphService(schema, device=dev)
svc.install_query(1, QueryPlan("u").out("click", 10).out("sim", 5))
rs = np.random.RandomState(0)
BATCH, NB = 200_000, 40
REC_BYTES = 8 + 8 + 8 + 4            # src, dst, ts, weight
# ---- ingest: record batches come from pinned host memory (the Kafka poller's role), one kernel launch applies a batch
batches = []
t = 0
for b in range(NB):
    et = "click" if b % 2 == 0 else "sim"
    src = torch.from_numpy(rs.zipf(1.3, BATCH).astype(np.int64) % (NU if et == "click" else NI)).pin_memory()
    dst = torch.from_numpy(rs.randint(0, NI, BATCH).astype(np.int64)).pin_memory()
    ts = torch.arange(t, t + BATCH, dtype=torch.int64).pin_memory(); t += BATCH
    w = torch.rand(BATCH).pin_memory()
    batches.append((et, src, dst, ts, w))
feat = torch.randn(NI, FD)
svc.apply_updates({"vertices": {"i": {"id": torch.arange(NI), "ts": torch.zeros(NI, dtype=torch.int64), "feat": feat}}})
for et, src, dst, ts, w in batches[:4]:
    svc.apply_updates({"edges": {et: {"src": src, "dst": dst, "ts": ts, "weight": w}}})
if dev == "cuda":
    torch.cuda.synchronize()
t0 = time.perf_counter()
for et, src, dst, ts, w in batches[4:]:
    svc.apply_updates({"edges": {et: {"src": src, "dst": dst, "ts": ts, "weight": w}}})
if dev == "cuda":
    torch.cuda.synchronize()
dt = time.perf_counter() - t0
n_rec = (NB - 4) * BATCH
ingest = {"records_per_s": n_rec / dt, "MB_per_s": n_rec * REC_BYTES / dt / 1e6, "batch_records": BATCH,
          "note": "zipf(1.3) sources (hot vertices), includes the pinned-host -> device copy of every batch"}
# ---- single-vertex 2-hop queries (the /infer?qid&vid path): wall-clock latency including the D2H of the answer
lat = []
qv = rs.randint(0, NU, 3000)
for i, v in enumerate(qv):
    t1 = time.perf_counter()
    res = svc.run_query(1, [int(v)])
    ids = res["hops"][1]["ids"].cpu()
    f = res["hops"][1]["features"].cpu()
    if i >= 200:
        lat.append((time.perf_counter() - t1) * 1e3)
lat = np.array(lat)
single = {"p50_ms": float(np.percentile(lat, 50)), "p99_ms": float(np.percentile(lat, 99)), "qps_single_thread": float(1e3 / lat.mean())}
# ---- batched queries (one launch per hop for the whole batch)
qps = {}
for B in (64, 1024, 16384):
    vs = torch.from_numpy(rs.randint(0, NU, (30, B)))
    for j in range(3):
        svc.run_query(1, vs[j])["hops"][1]["ids"].cpu()
    t1 = time.perf_counter()
    for j in range(3, 30):
        res = svc.run_query(1, vs[j])
        res["hops"][1]["ids"].cpu(); res["hops"][1]["features"].cpu()
    qps[str(B)] = 27 * B / (time.perf_counter() - t1)
out = {"what": "DGS (streaming TopK-by-timestamp sampler in HBM) on 1 x %s" % (torch.cuda.get_device_name(0) if dev == "cuda" else "cpu"),
       "reference_published": {"p99_ms": 20, "qps": 20000, "ingest_MB_per_s": 110, "hardware": "64 cores / 256 GB"},
       "ingest": ingest, "query_2hop_single": single, "query_2hop_batched_qps": qps,
       "vs_reference": {"ingest": ingest["MB_per_s"] / 110, "p99": 20 / single["p99_ms"], "qps_batched_1024": qps["1024"] / 20000}}
print(json.dumps(out))
