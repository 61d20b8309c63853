#!/usr/bin/env python
"""Fused GraphSAGE with batch normalisation of the hidden layers (``EgoGraphSAGE(batch_norm=True)``).

Graphs: bench.py's ``products_sage2`` (2.45 M nodes, 123.7 M edges, 100 bf16 features, fan-out 25,10) and ``sage3``
(ogbn-papers100M shape at 1/32 scale, 128 bf16 features, fan-out 15,10,5) shapes, hidden 256.  For each it runs the
supervised trainer (B = 1024 seeds) with BN off and on, and on the products shape the link trainer (B = 512 positive
edges, 5 random negatives, 64-wide embeddings) with BN off and on.  It reports
  - steps/s of the captured device-only step (CUDA events around K replays, fresh roots every replay),
  - the device time of every kernel of one replay (torch.profiler, mean over the profiled replays, as
    tools/bench_embed_sage.py),
  - for each BN kernel the bytes it must move per step, computed from the shapes (all BN layers together), and the
    achieved bytes/s against the H100 SXM's 3.35 TB/s.
The card name, power limit and max SM clock are printed in the same run.

    python tools/bench_sage_bn.py [--configs products_sage2 sage3] [--steps 1000] [--warmup 20] [--small]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

HBM_BPS = 3.35e12
HIDDEN, BATCH, LINK_BATCH, NEG, EMB = 256, 1024, 512, 5, 64
BN_KERNELS = ("bn_stats", "bn_apply", "bn_dY", "bn_bwd_sum", "bn_bwd_apply")


def bn_bytes(tr):
    """bytes each BN kernel must move in one step, summed over the BN layers: Z fp32, H / dY / dZ bf16; dY reads H,
    the self rows of dA of the layer above and (once per parent) its neighbour rows"""
    out = dict.fromkeys(BN_KERNELS, 0)
    for ly, up in zip(tr.layers[:-1], tr.layers[1:]):
        rc = ly.rows * ly.conv.out_dim
        self_rows = sum(up.offs[i + 1] - up.offs[i] for i in range(up.nseg))
        out["bn_stats"] += 4 * rc
        out["bn_apply"] += 4 * rc + 2 * rc
        out["bn_dY"] += 2 * rc + 2 * rc + 2 * 2 * self_rows * ly.conv.out_dim
        out["bn_bwd_sum"] += 2 * rc + 4 * rc
        out["bn_bwd_apply"] += 2 * rc + 4 * rc + 2 * rc
    return out


def key(name, seen, L):
    """per-kernel label: the BN kernels by their role, the rest as tools/step_timeline.py names them"""
    from step_timeline import label
    base = name.split("(")[0].replace("void ", "").replace("glb::", "")
    for k, v in (("bn_colsum_kernel<false>", "bn_stats"), ("bn_apply_kernel", "bn_apply"),
                 ("bn_colsum_kernel<true>", "bn_bwd_sum"), ("bn_bwd_apply_kernel", "bn_bwd_apply")):
        if base == k:
            return v
    if base.startswith("sage_bwd_dz_kernel"):
        return "bn_dY"
    return label(name, seen, L)


def time_and_profile(tr, roots, steps, warmup, replays):
    import torch
    from torch.profiler import ProfilerActivity, profile
    tr.capture()
    for i in range(warmup):
        tr.step_device(*roots(i))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        tr.step_device(*roots(warmup + i))
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(replays):
            tr.step_device(*roots(i))
        torch.cuda.synchronize()
    evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "glb::" in e.name],
                 key=lambda e: e.time_range.start)
    ends = [i for i, e in enumerate(evs) if "adam_pack" in e.name]
    per, n_rep = {}, 0
    for lo, hi in zip(ends[:-1], ends[1:]):
        seen = {}
        for e in evs[lo + 1:hi + 1]:
            k = key(e.name, seen, tr.L)
            per[k] = per.get(k, 0.0) + (e.time_range.end - e.time_range.start)
        n_rep += 1
    per = {k: v / max(n_rep, 1) for k, v in per.items()}
    return ms, per, n_rep


def report(name, cfg, ms, per, n_rep, moved):
    print("%s %s  steps/s %.0f  (%.1f us/step)" % (name, cfg, 1e3 / ms, ms * 1e3))
    print("  kernel us per replay (mean of %d): %s" % (n_rep, "  ".join("%s %.1f" % (k, v) for k, v in per.items())))
    if moved is None:
        return
    for k in BN_KERNELS:
        us, b = per.get(k, 0.0), moved[k]
        bps = b / (us * 1e-6) if us > 0 else 0.0
        print("  %s: %.1f MB in %.1f us = %.2f TB/s (%.0f %% of 3.35 TB/s)" % (k, b / 1e6, us, bps / 1e12, 100 * bps / HBM_BPS))


def main():
    import torch

    import bench
    import graphlearn_b200 as gl
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.synthetic import make_partitioned_sources
    from step_timeline import card

    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["products_sage2", "sage3"], choices=["products_sage2", "sage3"])
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--replays", type=int, default=6, help="profiled replays for the per-kernel times")
    ap.add_argument("--small", action="store_true", help="small graphs (functional check only)")
    a = ap.parse_args()
    rt = init()
    assert rt.is_cuda, "bench_sage_bn needs a CUDA device"
    print("card:", torch.cuda.get_device_name(0), "|", card())
    gl.set_feature_dtype("bf16")
    dev = rt.device
    for name in a.configs:
        cfg = bench.CONFIGS[name]
        shape, fan = dict(cfg["shape"]), cfg["fanouts"]
        if a.small:
            shape.update(num_nodes=200_000, num_edges=5_000_000)
        node_src, edge_src = make_partitioned_sources(rt, seed=0, **shape)
        g = gl.Graph()
        g.node(node_src, "n", decoder=gl.Decoder(labeled=True, attr_types=["float"] * shape["feat_dim"]))
        g.edge(edge_src, ("n", "n", "e"), decoder=gl.Decoder())
        g.init()
        del node_src, edge_src
        nodes, csr = g.store.nodes["n"], g.store.edges["e"]
        n, L = nodes.n_local, len(fan)
        total = a.warmup + a.steps + a.replays
        gen = torch.Generator(device=dev).manual_seed(1234)
        seeds = torch.randint(0, n, (total, BATCH), device=dev, generator=gen)
        pos = torch.randint(0, csr.n_edges, (total, LINK_BATCH), device=dev, generator=gen)
        src, dst = csr._row_of_edge[pos], csr.indices.local[pos]
        kinds = ("supervised", "link") if name == "products_sage2" else ("supervised",)
        for kind in kinds:
            for bn in (False, True):
                torch.manual_seed(0)
                if kind == "supervised":
                    m = EgoGraphSAGE(shape["feat_dim"], HIDDEN, shape["num_classes"], L, batch_norm=bn).to(dev)
                    tr = FastSageTrainer(rt, nodes, csr, m, fan, BATCH)
                    roots = lambda i: (seeds[i],)                           # noqa: E731
                else:
                    m = EgoGraphSAGE(shape["feat_dim"], HIDDEN, EMB, L, batch_norm=bn).to(dev)
                    tr = FastLinkSageTrainer.from_graph(g, "e", m, fan, LINK_BATCH, NEG)
                    roots = lambda i: (src[i], dst[i])                      # noqa: E731
                report("%s %s" % (name, kind), "bn=%s" % ("on" if bn else "off"),
                       *time_and_profile(tr, roots, a.steps, a.warmup, a.replays), bn_bytes(tr) if bn else None)
                del tr, m
                torch.cuda.synchronize()
                torch.cuda.empty_cache()
        del g, nodes, csr
    rt.shutdown()


if __name__ == "__main__":
    main()
