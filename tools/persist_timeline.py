"""Per-role clock64 trace of the persistent fused kernel (one launch of the flagship's layer 1 and of layer 2):
where a CTA's time goes - id staging, gather, MMA, epilogue - in cycles relative to the CTA start."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from graphlearn_b200.engine.fast_sage import FastSageTrainer
from graphlearn_b200.models.graphsage import EgoGraphSAGE
from graphlearn_b200.parallel.runtime import init, native
from graphlearn_b200.store.synthetic import make_sharded_graph

rt = init()
C = native()
nodes, csr = make_sharded_graph(rt, num_nodes=2_449_029, num_edges=123_718_280, feat_dim=100, num_classes=47, seed=0,
                                feature_dtype=torch.bfloat16)
model = EgoGraphSAGE(100, 256, 47, 2).to(rt.device)
tr = FastSageTrainer(rt, nodes, csr, model, [25, 10], 1024, use_cuda_graph=False)
g = torch.Generator().manual_seed(0)
for _ in range(3):
    tr.step(torch.randint(0, nodes.n_local, (1024,), generator=g))
torch.cuda.synchronize()
NAMES = {0: "start", 1: "W image ready", 2: "cta end"}
for i in range(4):
    NAMES[4 + 2 * i] = "mma+epi%d begin (A full)" % i; NAMES[5 + 2 * i] = "mma+epi%d end" % i
    NAMES[20 + 2 * i] = "stage%d begin" % i; NAMES[21 + 2 * i] = "stage%d end" % i
    NAMES[28 + 3 * i] = "gather%d ptrs ready" % i; NAMES[29 + 3 * i] = "gather%d items done (warp 7)" % i
    NAMES[30 + 3 * i] = "gather%d arrived" % i


def traced(fn, label):
    n_sm = torch.cuda.get_device_properties(rt.device).multi_processor_count
    buf = torch.zeros(n_sm * 64, dtype=torch.int64, device=rt.device)
    C.sage_set_debug_trace(buf)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(); fn(); ev1.record()
    torch.cuda.synchronize()
    C.sage_set_debug_trace(None)
    t = buf.view(n_sm, 64).cpu()
    print("==== %s: %.1f us (CUDA events)" % (label, ev0.elapsed_time(ev1) * 1e3))
    for cta in (0, 1, n_sm // 2, n_sm - 1):
        row = t[cta]
        if int(row[0]) == 0:
            continue
        evs = sorted((int(row[i]) - int(row[0]), NAMES[i]) for i in NAMES if int(row[i]) != 0)
        print("  CTA %d:" % cta)
        for c, n in evs:
            print("    %8d cyc  %s" % (c, n))
    live = t[:, 60] != 0
    g0, g1 = t[live, 60], t[live, 62]
    print("  globaltimer: first CTA entry -> last CTA exit %.1f us; CTA entry spread %.1f us; per-CTA (exit-entry) median %.1f us; "
          "entry->start (init) median %d cyc" % ((int(g1.max()) - int(g0.min())) / 1e3, (int(g0.max()) - int(g0.min())) / 1e3,
                                                float((g1 - g0).float().median()) / 1e3, int((t[live, 0] - t[live, 61]).median())))
    ends = (t[:, 2] - t[:, 0])[t[:, 0] != 0]
    print("  CTA lifetime cycles: min %d median %d max %d" % (int(ends.min()), int(ends.median()), int(ends.max())))


# one eager step, the two forward launches traced separately via a hook on the native call
orig = C.sage_fused_multi
calls = []
def hook(*a):
    calls.append(a)
    return orig(*a)
tr.C = type("P", (), {"__getattr__": lambda self, n: hook if n == "sage_fused_multi" else getattr(C, n)})()
tr.step(torch.randint(0, nodes.n_local, (1024,), generator=g))
torch.cuda.synchronize()
for i, a in enumerate(calls[:3]):
    for rep in range(2):
        traced(lambda: orig(*a), "persistent launch %d (rep %d)" % (i + 1, rep))
# dW kernel launches of one eager step, re-run as they ran
dw_calls = []
orig_dw = C.sage_bwd_dw
def hook_dw(*a, **kw):
    dw_calls.append((a, kw))
    return orig_dw(*a, **kw)
tr.C = type("P", (), {"__getattr__": lambda self, n: hook_dw if n == "sage_bwd_dw" else getattr(C, n)})()
tr._skip_opt = True
tr.step(torch.randint(0, nodes.n_local, (1024,), generator=g))
torch.cuda.synchronize()
for a, kw in dw_calls:
    ts = []
    for rep in range(5):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(); orig_dw(*a, **kw); ev1.record(); torch.cuda.synchronize()
        ts.append(ev0.elapsed_time(ev1) * 1e3)
    print("dW launch rows=%d: %s us" % ((a[10] if len(a) > 10 else kw["a"]).size(0), ["%.1f" % x for x in ts]))
