#!/usr/bin/env python
"""Fused GraphSAGE with 257-512-wide layer inputs (split-K layers: the self half's launch, then the neighbour half's).

Graph: bench.py's ``products_sage2`` shape (2.45 M nodes, 123.7 M edges, fan-out 25,10, B = 1024 seeds) with F bf16
features.  Configurations: F = 300 and 500 with hidden 256 (layer 1 split), and F = 100 with hidden 512 (the top layer
reads a 512-wide input and is split).  For each it reports
  - steps/s of the fused trainer's captured device-only step (CUDA events around K replays, fresh roots every replay),
  - steps/s of the autograd ``SageTrainer`` on the same model, graph and batches (eager, synchronised every step),
  - the device time of each forward launch of one replay (torch.profiler, mean over the profiled replays) and, for the
    two halves of a split layer, the feature and A bytes they must move (computed from the shapes) and the achieved
    bytes/s against the H100 SXM's 3.35 TB/s,
  - the time of one ``infer_all`` (layer-wise inference over every node, CUDA events, after one warm-up call).
The card name, power limit and max SM clock are printed in the same run.

    python tools/bench_sage_wide.py [--configs 300x256 500x256 100x512] [--steps 1000] [--warmup 20] [--small]
"""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

HBM_BPS = 3.35e12
BATCH = 1024


def launch_labels(tr):
    """labels of the step's forward launches in issue order"""
    out = []
    for l, ly in enumerate(tr.layers, 1):
        out += ["L%d_self" % l, "L%d_nbr" % l] if ly.split else ["L%d" % l]
    return out


def half_bytes(tr, ly):
    """bytes the two halves of split layer `ly` must move: bf16 self / neighbour rows read, bf16 A halves written (and
    the fp32 partial written by the self half and read by the neighbour half)"""
    d = ly.conv.in_self
    self_rows = sum(ly.fwd[2])
    nbr_rows = sum(m * k for m, k in zip(ly.fwd[2], ly.fwd[3]))
    kp, part = ly.kt // 2, ly.rows * ly.ns * ly.N * 4
    return {"self": 2 * d * self_rows + 2 * kp * ly.rows + part, "nbr": 2 * d * nbr_rows + 2 * kp * ly.rows + part}


def time_fused(tr, roots, steps, warmup, replays):
    import torch
    from torch.profiler import ProfilerActivity, profile
    tr.capture()
    for i in range(warmup):
        tr.step_device(roots(i))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        tr.step_device(roots(warmup + i))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(replays):
            tr.step_device(roots(i))
        torch.cuda.synchronize()
    evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "sage_persist_kernel" in e.name],
                 key=lambda e: e.time_range.start)
    labels = launch_labels(tr)
    per = dict.fromkeys(labels, 0.0)
    n_rep = len(evs) // len(labels)
    for i, e in enumerate(evs[:n_rep * len(labels)]):
        per[labels[i % len(labels)]] += e.time_range.end - e.time_range.start
    return ms, {k: v / max(n_rep, 1) for k, v in per.items()}, n_rep


def time_autograd(rt, nodes, csr, model, fan, seeds, steps):
    import torch
    from graphlearn_b200.engine.trainer import SageTrainer
    tr = SageTrainer(rt, nodes, csr, model, fan, BATCH, use_cuda_graph=False)
    for i in range(3):
        tr.step(seeds[i].cpu())
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        tr.step(seeds[3 + i].cpu())
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


def time_infer(tr):
    import torch
    tr.infer_all()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    tr.infer_all()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    import torch

    import bench
    import graphlearn_b200 as gl
    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.synthetic import make_partitioned_sources
    from step_timeline import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["300x256", "500x256", "100x512"],
                    help="FEATURESxHIDDEN, each in 1..512")
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--autograd-steps", type=int, default=50)
    ap.add_argument("--replays", type=int, default=6, help="profiled replays for the per-launch times")
    ap.add_argument("--small", action="store_true", help="small graph (functional check only)")
    a = ap.parse_args()
    rt = init()
    assert rt.is_cuda, "bench_sage_wide needs a CUDA device"
    print("card:", torch.cuda.get_device_name(0), "|", card())
    gl.set_feature_dtype("bf16")
    dev = rt.device
    cfg = bench.CONFIGS["products_sage2"]
    fan = cfg["fanouts"]
    for c in a.configs:
        feat, hidden = (int(x) for x in c.split("x"))
        shape = dict(cfg["shape"], feat_dim=feat)
        if a.small:
            shape.update(num_nodes=200_000, num_edges=5_000_000)
        node_src, edge_src = make_partitioned_sources(rt, seed=0, **shape)
        g = gl.Graph()
        g.node(node_src, "n", decoder=gl.Decoder(labeled=True, attr_types=["float"] * feat))
        g.edge(edge_src, ("n", "n", "e"), decoder=gl.Decoder())
        g.init()
        del node_src, edge_src
        nodes, csr = g.store.nodes["n"], g.store.edges["e"]
        total = a.warmup + a.steps + a.replays
        seeds = torch.randint(0, nodes.n_local, (total, BATCH), device=dev, generator=torch.Generator(device=dev).manual_seed(1234))
        torch.manual_seed(0)
        m = EgoGraphSAGE(feat, hidden, shape["num_classes"], len(fan)).to(dev)
        tr = FastSageTrainer(rt, nodes, csr, m, fan, BATCH)
        ms, per, n_rep = time_fused(tr, lambda i: seeds[i], a.steps, a.warmup, a.replays)
        print("products %s: fused %.0f steps/s (%.1f us/step); split layers %s" % (
            c, 1e3 / ms, ms * 1e3, [l for l, ly in enumerate(tr.layers, 1) if ly.split]))
        print("  forward launch us per replay (mean of %d): %s" % (n_rep, "  ".join("%s %.1f" % kv for kv in per.items())))
        for l, ly in enumerate(tr.layers, 1):
            if ly.split:
                for half, b in half_bytes(tr, ly).items():
                    us = per["L%d_%s" % (l, half)]
                    bps = b / (us * 1e-6) if us > 0 else 0.0
                    print("  L%d %s half: %.1f MB in %.1f us = %.2f TB/s (%.0f %% of 3.35 TB/s)" % (
                        l, half, b / 1e6, us, bps / 1e12, 100 * bps / HBM_BPS))
        print("  infer_all %.1f ms" % time_infer(tr))
        del tr
        torch.cuda.synchronize()
        torch.manual_seed(0)
        m2 = EgoGraphSAGE(feat, hidden, shape["num_classes"], len(fan)).to(dev)
        ams = time_autograd(rt, nodes, csr, m2, fan, seeds, a.autograd_steps)
        print("  autograd SageTrainer %.0f steps/s (%.1f us/step)" % (1e3 / ams, ams * 1e3))
        del m, m2, g, nodes, csr
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    rt.shutdown()


if __name__ == "__main__":
    main()
