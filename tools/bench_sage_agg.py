"""Speed of the fused GraphSAGE engine per aggregator (mean, sum, max, gcn) and dropout rate on the headline workload.

For each aggregator and dropout rate it builds the `products_sage2` trainer exactly as bench.py does (gl.Graph -> GSL
query -> FastSageTrainer.from_query, bf16 feature rows) around ``EgoGraphSAGE(..., agg_type=a, dropout=p)`` and reports
  - steps/s of the captured step (bench.time_trainer's device-timed region),
  - the device time of every kernel of one replay (torch.profiler, mean over the profiled replays),
  - ``infer_all`` in ms (CUDA events, after a warm-up call).
The card name, power limit and max SM clock are printed in the same run.

    python tools/bench_sage_agg.py [--agg mean max gcn] [--dropout 0 0.5] [--steps 1000] [--warmup 20] [--small]
"""
import argparse
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from graphlearn_b200.models import graphsage
    from graphlearn_b200.parallel.runtime import init
    from step_timeline import card, label

    ap = argparse.ArgumentParser()
    ap.add_argument("--agg", nargs="+", default=["mean", "sum", "max", "gcn"], choices=["mean", "sum", "max", "gcn"])
    ap.add_argument("--dropout", nargs="+", type=float, default=[0.0], help="dropout rates between the layers")
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--replays", type=int, default=6, help="profiled replays for the per-kernel times")
    ap.add_argument("--small", action="store_true", help="small graph (functional check only)")
    a = ap.parse_args()
    rt = init()
    assert rt.is_cuda, "bench_sage_agg needs a CUDA device"
    print("card:", torch.cuda.get_device_name(0), "|", card())
    args = argparse.Namespace(cfg=bench.CONFIGS["products_sage2"], api="gsl", batch=bench.BATCH, engine="fast",
                              allreduce="peer", no_graph=False, warmup=a.warmup)
    shape = dict(args.cfg["shape"])
    if a.small:
        shape = dict(num_nodes=200_000, num_edges=5_000_000, feat_dim=100, num_classes=47)
    base = graphsage.EgoGraphSAGE
    for agg, drop in [(x, q) for x in a.agg for q in a.dropout]:
        # bench.build_trainer constructs graphsage.EgoGraphSAGE(in, hidden, classes, layers): give it the aggregator and
        # the dropout rate
        graphsage.EgoGraphSAGE = lambda *p, _agg=agg, _drop=drop, **kw: base(*p, agg_type=_agg, dropout=_drop, **kw)
        try:
            tr, nodes, _, _, _, g = bench.build_trainer(args, rt, shape, "bf16", 0)
        finally:
            graphsage.EgoGraphSAGE = base
        assert all(c.agg_type == agg for c in tr.convs) and tr.dropout == drop
        ms_dev = bench.time_trainer(args, rt, tr, nodes, a.steps)[0]
        sps = a.steps / (ms_dev / 1e3)
        # per-kernel device time of the captured step
        seeds = torch.randint(0, nodes.n_local, (a.replays, args.batch), device=rt.device)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for i in range(a.replays):
                tr.step_device(seeds[i])
            torch.cuda.synchronize()
        evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "glb::" in e.name],
                     key=lambda e: e.time_range.start)
        ends = [i for i, e in enumerate(evs) if "adam_pack" in e.name]
        per, n_rep = {}, 0
        for lo, hi in zip(ends[:-1], ends[1:]):             # whole replays: after one adam_pack up to the next
            seen = {}
            for e in evs[lo + 1:hi + 1]:
                k = label(e.name, seen, tr.L)
                per[k] = per.get(k, 0.0) + (e.time_range.end - e.time_range.start)
            n_rep += 1
        # layer-wise full-neighbourhood inference
        tr.infer_all()
        torch.cuda.synchronize()
        t_inf = []
        for _ in range(3):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            tr.infer_all()
            e1.record()
            torch.cuda.synchronize()
            t_inf.append(e0.elapsed_time(e1))
        print("agg=%s dropout=%g  steps/s %.0f  (%d steps, %.1f us/step)  infer_all ms %s" %
              (agg, drop, sps, a.steps, ms_dev * 1e3 / a.steps, " / ".join("%.2f" % t for t in t_inf)))
        print("  kernel us per replay (mean of %d): %s" %
              (n_rep, "  ".join("%s %.1f" % (k, v / max(n_rep, 1)) for k, v in per.items())))
        del tr, nodes, g
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    rt.shutdown()


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    main()
