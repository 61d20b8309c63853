#!/usr/bin/env python
"""Unsupervised (link-prediction) GraphSAGE: the captured step of ``FastLinkSageTrainer`` against the autograd path of
``examples/train_unsupervised_sage.py`` (GSL edge query with ``outNeg`` + dense EgoGraphSAGE + nn/loss.py + Adam),
same objective, same graph, same shapes.

    python tools/bench_link_sage.py [--steps 500] [--autograd-steps 50] [--small]

Graph: bench.py's ogbn-products shape (2.45 M nodes, 123.7 M edges, 100-d features), fan-out [25, 10], hidden 256,
embedding 64, B = 512 positive edges and 5 random negatives per step, sigmoid loss.  Prints one JSON line with the
card name and power limit read in the same run.  Nothing is written.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PRODUCTS = dict(num_nodes=2_449_029, num_edges=123_718_280, feat_dim=100, num_classes=47)
FANOUTS, HIDDEN, EMB, BATCH, NEG = [25, 10], 256, 64, 512, 5


def card():
    import torch
    info = {"name": torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [p.strip() for p in out.split(",")[:2]]
    except Exception as e:              # the number is still printed, without the limit
        info["power_limit"] = "unknown (%r)" % (e,)
    return info


def count_launches(tr, src, dst):
    """kernel launches of one eager end-to-end step (edge staging included), ours (glb::) vs library kernels"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    graph, tr.graph = tr.graph, None
    try:
        with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
            tr.step(src, dst)
            torch.cuda.synchronize()
    finally:
        tr.graph = graph
    own, lib, names = 0, 0, {}
    for ev in prof.events():
        if ev.device_type is not None and str(ev.device_type).endswith("CUDA") and ev.name and \
                not ev.name.startswith("Memcpy") and not ev.name.startswith("Memset"):
            if "glb::" in ev.name:
                own += 1
                key = ev.name.split("(")[0][:60]
                names[key] = names.get(key, 0) + 1
            else:
                lib += 1
    return own, lib, names


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--autograd-steps", type=int, default=50)
    ap.add_argument("--small", action="store_true", help="200 k nodes / 5 M edges, for quick functional runs")
    a = ap.parse_args()

    import torch

    import graphlearn_b200 as gl
    from graphlearn_b200 import models
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.nn.data import Data
    from graphlearn_b200.nn.loss import sigmoid_cross_entropy_loss
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.synthetic import make_partitioned_sources
    rt = init()
    if not rt.is_cuda:
        raise SystemExit("bench_link_sage.py needs a CUDA device")
    shape = dict(PRODUCTS)
    if a.small:
        shape.update(num_nodes=200_000, num_edges=5_000_000)
    dev = rt.device
    t0 = time.time()
    node_src, edge_src = make_partitioned_sources(rt, seed=0, **shape)
    node_src.pop("labels")              # the link objective needs none
    g = gl.Graph()
    g.node(node_src, "n", decoder=gl.Decoder(attr_types=["float"] * shape["feat_dim"]))
    g.edge(edge_src, ("n", "n", "e"), decoder=gl.Decoder())
    g.init()
    del node_src, edge_src
    torch.cuda.synchronize()
    build_s = time.time() - t0
    csr = g.store.edges["e"]

    # ---- engine: captured link step, device timed, fresh edges every replay
    torch.manual_seed(0)
    model = models.EgoGraphSAGE(shape["feat_dim"], HIDDEN, EMB, 2).to(dev)
    tr = FastLinkSageTrainer.from_graph(g, "e", model, FANOUTS, BATCH, NEG, lr=3e-3)
    total = a.warmup + a.steps + 4
    gen = torch.Generator(device=dev).manual_seed(1234)
    pos = torch.randint(0, csr.n_edges, (total, BATCH), device=dev, generator=gen)
    src = csr._row_of_edge[pos] * rt.world + rt.rank
    dst = csr.indices.local[pos]
    tr.capture()
    for i in range(a.warmup):
        tr.step_device(src[i], dst[i])
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record()
    for i in range(a.steps):
        tr.step_device(src[a.warmup + i], dst[a.warmup + i])
    ev1.record()
    torch.cuda.synchronize()
    ms_dev = ev0.elapsed_time(ev1) / a.steps
    # end to end: host edge traversal (step_edges) -> pinned staging -> step graph -> loss to the host
    for _ in range(3):
        tr.step_edges()
    torch.cuda.synchronize()
    ev2, ev3 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev2.record()
    done = 0
    while done < a.steps:
        try:
            last = tr.step_edges()
        except gl.OutOfRangeError:
            continue
        done += 1
    ev3.record()
    torch.cuda.synchronize()
    ms_e2e = ev2.elapsed_time(ev3) / a.steps
    engine_loss = float(last)
    own, lib, names = count_launches(tr, src[0].cpu(), dst[0].cpu())
    del tr
    torch.cuda.empty_cache()

    # ---- autograd path of examples/train_unsupervised_sage.py on the same graph and shapes
    def ego(node, prefix):
        node.outV("e").sample(FANOUTS[0]).by("random").alias(prefix + "1") \
            .outV("e").sample(FANOUTS[1]).by("random").alias(prefix + "2")
    e = g.E("e").batch(BATCH).shuffle(traverse=True).alias("edge")
    s = e.outV().alias("s"); ego(s, "s")
    d = e.inV().alias("d"); ego(d, "d")
    n = s.outNeg("e").sample(NEG).by("random").alias("n"); ego(n, "n")
    ds = gl.Dataset(e.values())
    torch.manual_seed(0)
    model2 = models.EgoGraphSAGE(shape["feat_dim"], HIDDEN, EMB, 2).to(dev)
    opt = torch.optim.Adam(model2.parameters(), lr=3e-3)

    def f(v):
        return Data.from_values(v).floats

    def enc(r, p):
        return model2([f(r[p]), f(r[p + "1"]), f(r[p + "2"])], FANOUTS)

    def ag_step():
        while True:
            try:
                r = ds.next()
                break
            except gl.OutOfRangeError:
                continue
        zs, zd, zn = enc(r, "s"), enc(r, "d"), enc(r, "n")
        pos_ = (zs * zd).sum(-1)
        neg_ = (zs.unsqueeze(1) * zn.view(zs.size(0), NEG, -1)).sum(-1)
        loss = sigmoid_cross_entropy_loss(pos_, neg_.reshape(-1))
        opt.zero_grad(); loss.backward(); opt.step()
        return loss.detach()
    for _ in range(3):
        ag_step()
    torch.cuda.synchronize()
    ev4, ev5 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev4.record()
    for _ in range(a.autograd_steps):
        ag_loss = ag_step()
    ev5.record()
    torch.cuda.synchronize()
    ms_ag = ev4.elapsed_time(ev5) / a.autograd_steps

    print(json.dumps({
        "metric": "unsupervised GraphSAGE link-prediction train steps/s (2 layers, fan-out 25,10, hidden 256, emb 64, "
                  "B=512 edges + 5 random negatives each, sigmoid loss)",
        "card": card(), "n_gpus": rt.world,
        "graph": {"num_nodes": shape["num_nodes"], "num_edges": shape["num_edges"], "feat_dim": shape["feat_dim"],
                  "build_s": round(build_s, 1)},
        "roots_per_step": BATCH * (2 + NEG),
        "engine": {"steps_per_s": 1e3 / ms_dev, "ms_per_step": ms_dev, "e2e_steps_per_s": 1e3 / ms_e2e,
                   "e2e_ms_per_step": ms_e2e, "steps": a.steps, "final_loss": engine_loss,
                   "own_kernels_per_step": own, "library_kernels_per_step": lib, "own_kernel_names": names},
        "autograd": {"steps_per_s": 1e3 / ms_ag, "ms_per_step": ms_ag, "steps": a.autograd_steps,
                     "final_loss": float(ag_loss),
                     "path": "GSL E().outNeg() query -> interpreter -> dense EgoGraphSAGE autograd -> torch Adam"},
        "speedup": ms_ag / ms_dev,
    }))
    rt.shutdown()


if __name__ == "__main__":
    main()
