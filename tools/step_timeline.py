"""Device timeline of one captured training step of the headline workload (bench.py products_sage2, 1 GPU).

Builds the trainer exactly as bench.py does (gl.Graph -> GSL query -> FastSageTrainer.from_query, bf16 feature rows),
captures and warms it up, then profiles a few ``step_device`` replays with torch.profiler (CUPTI reports the kernels
inside graph replays).  For one replay it prints every kernel with its device start, end and stream in start order, the
main-chain critical path with the idle gap before each of its kernels, and whether a sampling kernel overlaps the start
of the layer-1 forward.  The card name, power limit and max SM clock are printed in the same run.

    python tools/step_timeline.py [--config products_sage2] [--replays 6] [--small]
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = "name,power.limit,clocks.max.sm"
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=10).stdout.strip()
    except Exception as e:          # no nvidia-smi: still print the device name torch sees
        return "nvidia-smi unavailable (%s)" % e


def label(name, seen, L):
    """stable short name; the launches of one kernel in a step are told apart by their order: the persistent kernel runs
    the forward L1..L<L>, the backward runs dA<L>..dA2 and dW<L>..dW1"""
    base = name.split("(")[0].replace("void ", "").replace("glb::", "")
    base = base.split("<")[0]
    i = seen.get(base, 0)
    seen[base] = i + 1
    if base == "sage_persist_kernel":
        return "L%d" % (i + 1)
    if base == "sage_bwd_da_kernel":
        return "dA%d" % (L - i)
    if base == "sage_bwd_dw_kernel":
        return "dW%d" % (L - i)
    if base == "sample_neighbors_kernel":
        return "sample_hop%d" % (i + 1)
    return base


def main():
    import torch
    from torch.profiler import ProfilerActivity, profile

    import bench
    from graphlearn_b200.parallel.runtime import init

    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="products_sage2", choices=["products_sage2", "sage3"])
    ap.add_argument("--replays", type=int, default=6)
    ap.add_argument("--small", action="store_true", help="small graph (functional check only)")
    a = ap.parse_args()
    rt = init()
    assert rt.is_cuda, "step_timeline needs a CUDA device"
    print("card:", torch.cuda.get_device_name(0), "|", card())
    args = argparse.Namespace(cfg=bench.CONFIGS[a.config], api="gsl", batch=bench.BATCH, engine="fast", allreduce="peer",
                              no_graph=False)
    shape = dict(args.cfg["shape"])
    if a.small:
        shape = dict(num_nodes=200_000, num_edges=5_000_000, feat_dim=100, num_classes=47)
    tr, nodes, _, _, _, _ = bench.build_trainer(args, rt, shape, "bf16", 0)
    n = nodes.n_local
    seeds = torch.randint(0, n, (64 + a.replays, args.batch), device=rt.device)
    tr.seeds.copy_(seeds[0])
    tr.capture()
    for i in range(40):
        tr.step_device(seeds[i + 1])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(a.replays):
            tr.step_device(seeds[41 + i])
        torch.cuda.synchronize()
    evs = sorted([e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "glb::" in e.name],
                 key=lambda e: e.time_range.start)
    # one replay = the kernels after one adam_pack up to and including the next one; take the second-to-last replay
    ends = [i for i, e in enumerate(evs) if "adam_pack" in e.name]
    assert len(ends) >= 3, "too few replays in the trace"
    lo, hi = ends[-3] + 1, ends[-2] + 1
    rep = evs[lo:hi]
    t0 = rep[0].time_range.start
    seen = {}
    rows = []
    for e in rep:
        rows.append((label(e.name, seen, tr.L), e.time_range.start - t0, e.time_range.end - t0, getattr(e, "device_resource_id", None)))
    print("replay: %d kernels, first start -> adam_pack end %.1f us; adam_pack end to end of the next %.1f us" %
          (len(rep), rows[-1][2], evs[ends[-2]].time_range.end - evs[ends[-3]].time_range.end))
    print("%-18s %9s %9s %8s  %s" % ("kernel", "start us", "end us", "dur us", "stream"))
    for name, s, e, st in rows:
        print("%-18s %9.1f %9.1f %8.1f  %s" % (name, s, e, e - s, st))
    # main chain: previous replay's adam_pack -> L1 .. L<L> (-> softmax_ce) -> dA<L> -> dW<L-1> -> dA<L-1> .. dA2 -> dW1
    # -> adam_pack (dW<L> runs beside dA<L>)
    L = tr.L
    order = ["L%d" % l for l in range(1, L + 1)] + ["softmax_ce_kernel"]
    order += [n for l in range(L, 1, -1) for n in ("dA%d" % l, "dW%d" % (l - 1))] + ["adam_pack_kernel"]
    chain = [n for n in order if any(r[0] == n for r in rows)]
    by = {r[0]: r for r in rows}
    prev_end = evs[ends[-3]].time_range.end - t0
    busy = gaps = 0.0
    print("critical path (main chain):")
    for n in chain:
        _, s, e, _ = by[n]
        print("  %-18s gap before %6.1f us   kernel %6.1f us" % (n, s - prev_end, e - s))
        gaps += s - prev_end
        busy += e - s
        prev_end = e
    print("  sum: kernels %.1f us + gaps %.1f us = %.1f us" % (busy, gaps, busy + gaps))
    l1s = by["L1"][1]
    ov = [r for r in rows if r[0].startswith("sample") and r[1] <= l1s + 5.0 and r[2] > l1s]
    print("sampling kernels overlapping the first 5 us of L1:", ", ".join("%s (%.1f-%.1f)" % (r[0], r[1], r[2]) for r in ov) or "none")
    rt.shutdown()


if __name__ == "__main__":
    main()
