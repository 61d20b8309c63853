#!/usr/bin/env python
"""Fused GraphSAGE with a learned input embedding (``learn_input_embedding=True``).

Graph: bench.py's ogbn-products shape (2.45 M nodes, 123.7 M edges, 47 classes), hidden 256, bf16 learned table E of
width d.  Without ``--features`` the graph has no float attributes and E is layer 1's whole input.  With
``--features F`` it keeps F bf16 float attributes and every fan-out runs three configurations:
  - x       : the attributes alone, flag off, in_dim = F;
  - E+x     : the attributes and a d-wide E, in_dim = d + F (dA_1 over E's column blocks only);
  - E+x/fullA: the same with dA_1 over every column block (what the step would cost without the column windows).
For the supervised trainer (B = 1024 seeds) and the link trainer (B = 512 positive edges, 5 random negatives, 64-wide
embeddings) it reports
  - steps/s of the captured device-only step (CUDA events around K replays, fresh roots every replay),
  - the device time of every kernel of one replay (torch.profiler, mean over the profiled replays, as
    tools/bench_sage_agg.py),
  - for embed_grad_scatter and embed_lazy_adam: the bytes they must move, computed from the shapes and the touched-row
    count of the last timed step (unique valid ids of its hop buffers), and the achieved bytes/s against the H100 SXM's
    3.35 TB/s; the bytes dA_1 writes.
The card name, power limit and max SM clock are printed in the same run.  A 64-wide bf16 row fits fan-outs up to 15 in
the fused kernel's gather scratch (ops.sage.fused_supported), so without attributes d = 64 runs fan-out [15, 10] and
d = 128 the headline [25, 10]; with attributes every width here fits both.

    python tools/bench_embed_sage.py [--dims 64 128] [--features F] [--steps 1000] [--warmup 20] [--small]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

HBM_BPS = 3.35e12
HIDDEN, BATCH, LINK_BATCH, NEG, EMB = 256, 1024, 512, 5, 64
FANOUTS = {64: [15, 10], 128: [25, 10]}
FEATURE_FANOUTS = ([15, 10], [25, 10])


def moved_bytes(tr):
    """(scatter bytes, lazy Adam bytes, dA_1 bytes written, touched rows, layer-1 row reads) of the step whose hops are
    in tr._hops[...]"""
    import torch
    e, ly = tr.emb, tr.layers[0]
    hops = tr._hops[(tr._steps - 1) & 1]
    n, dp = e.master.size(0), e.master.size(1)
    ids = torch.cat(hops)
    touched = int(torch.unique(ids[(ids >= 0) & (ids < n)]).numel())
    items = sum(tr.n[:ly.nseg])
    reads = sum(m * (1 + k) for m, k in zip(tr.n[:ly.nseg], tr.fanouts[:ly.nseg]))
    amax = items * dp if ly.argmax is not None else 0
    # scatter: both halves of a dA_1 row (bf16) + the ids + argmax bytes in, one fp32 reduction per (row read, column)
    scatter = items * 2 * dp * 2 + reads * 8 + amax + reads * dp * 4
    # lazy Adam: the bitmap, and per touched row w, m, v, grad in and w, m, v, zeroed grad out (fp32) + the bf16 row
    adam = (n + 31) // 32 * 4 + touched * dp * (8 * 4 + 2)
    cols = sum(64 * (hi - lo) for lo, hi in ly.da_blocks) if ly.da_blocks else ly.kt
    return scatter, adam, ly.rows * cols * 2, touched, reads


def time_and_profile(tr, roots, steps, warmup, replays):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from step_timeline import label
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
    moved = moved_bytes(tr) if tr.emb is not None else None
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
            k = label(e.name, seen, tr.L)
            per[k] = per.get(k, 0.0) + (e.time_range.end - e.time_range.start)
        n_rep += 1
    per = {k: v / max(n_rep, 1) for k, v in per.items()}
    return ms, per, n_rep, moved


def report(name, cfg, fan, ms, per, n_rep, moved):
    print("%s %s fanouts=%s  steps/s %.0f  (%.1f us/step)" % (name, cfg, fan, 1e3 / ms, ms * 1e3))
    print("  kernel us per replay (mean of %d): %s" % (n_rep, "  ".join("%s %.1f" % (k, v) for k, v in per.items())))
    if moved is None:
        return
    sc_b, ad_b, da_b, touched, reads = moved
    print("  layer-1 row reads %d, touched rows %d, dA1 writes %.1f MB" % (reads, touched, da_b / 1e6))
    for k, b in (("embed_grad_scatter_kernel", sc_b), ("embed_lazy_adam_kernel", ad_b)):
        us = per.get(k, 0.0)
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
    ap.add_argument("--dims", nargs="+", type=int, default=None,
                    help="widths d of E (default: 64 128 without --features, 64 with it)")
    ap.add_argument("--features", type=int, default=0,
                    help="F > 0: keep F bf16 float attributes and compare x alone, E+x and E+x with a full dA_1")
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--replays", type=int, default=6, help="profiled replays for the per-kernel times")
    ap.add_argument("--small", action="store_true", help="small graph (functional check only)")
    a = ap.parse_args()
    F = a.features
    dims = a.dims or ([64] if F else [64, 128])
    if not F and any(d not in FANOUTS for d in dims):
        ap.error("without --features, --dims takes %s" % sorted(FANOUTS))
    rt = init()
    assert rt.is_cuda, "bench_embed_sage needs a CUDA device"
    print("card:", torch.cuda.get_device_name(0), "|", card())
    shape = dict(bench.CONFIGS["products_sage2"]["shape"])
    if a.small:
        shape.update(num_nodes=200_000, num_edges=5_000_000)
    shape["feat_dim"] = max(F, 1)
    node_src, edge_src = make_partitioned_sources(rt, seed=0, **shape)
    g = gl.Graph()
    if F:
        gl.set_feature_dtype("bf16")
        g.node(node_src, "n", decoder=gl.Decoder(labeled=True, attr_types=["float"] * F))
    else:
        node_src.pop("float_attrs")
        g.node(node_src, "n", decoder=gl.Decoder(labeled=True))
    g.edge(edge_src, ("n", "n", "e"), decoder=gl.Decoder())
    g.init()
    del node_src, edge_src
    nodes, csr = g.store.nodes["n"], g.store.edges["e"]
    assert nodes.float_dim == F and (not F or nodes.feats.local.dtype == torch.bfloat16)
    dev, n = rt.device, nodes.n_local
    total = a.warmup + a.steps + a.replays
    gen = torch.Generator(device=dev).manual_seed(1234)
    seeds = torch.randint(0, n, (total, BATCH), device=dev, generator=gen)
    pos = torch.randint(0, csr.n_edges, (total, LINK_BATCH), device=dev, generator=gen)
    src, dst = csr._row_of_edge[pos], csr.indices.local[pos]

    def run(kind, cfg, width, fan, flag, full_da=False):
        torch.manual_seed(0)
        if kind == "supervised":
            tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(width, HIDDEN, shape["num_classes"], 2).to(dev), fan, BATCH,
                                 learn_input_embedding=flag)
            roots = lambda i: (seeds[i],)                                   # noqa: E731
        else:
            tr = FastLinkSageTrainer.from_graph(g, "e", EgoGraphSAGE(width, HIDDEN, EMB, 2).to(dev), fan, LINK_BATCH, NEG,
                                                learn_input_embedding=flag)
            roots = lambda i: (src[i], dst[i])                              # noqa: E731
        if full_da:
            tr.layers[0].da_blocks = ()
        report(kind, cfg, fan, *time_and_profile(tr, roots, a.steps, a.warmup, a.replays))
        del tr
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    for d in dims:
        for kind in ("supervised", "link"):
            if not F:
                run(kind, "d=%d" % d, d, FANOUTS[d], True)
                continue
            for fan in FEATURE_FANOUTS:
                run(kind, "x (F=%d)" % F, F, fan, False)
                run(kind, "E+x (d=%d, F=%d)" % (d, F), d + F, fan, True)
                run(kind, "E+x/fullA (d=%d, F=%d)" % (d, F), d + F, fan, True, full_da=True)
    rt.shutdown()


if __name__ == "__main__":
    main()
