#!/usr/bin/env python
"""Layer-wise full-neighbourhood inference of a 2-layer GraphSAGE (100 -> 256 -> 47, mean; bench.py's model) over
every node of a products-shaped graph (2.45 M nodes, 123.7 M edges, bf16 features).

    python tools/bench_sage_inference.py [--reps 5] [--sampled-nodes 131072] [--small]

Measured, device time after warm-up:
  fused      ``FastSageTrainer.infer_all()``: one CSR-mode fused launch per layer (+ the hub pre-pass)
  composed   the same model through the existing kernels: per layer ``gather_agg`` (ragged, over the CSR) -> bf16
             ``[self || agg]`` -> ``tc_linear_forward``, on the same bf16 table
  sampled    the sampled ``predict`` loop in batches of 1024 on the first --sampled-nodes nodes (rate on that subset)
  skew       ``infer_all`` on the same node / edge counts with uniform degrees (skew=0) and heavier hubs (skew=2)
Gathered rows = self + neighbour rows of every layer; gathered GB/s counts their feature bytes (d x 2 B).  Prints one
JSON line with the card name, power limit and max SM clock read in the same run.  Nothing is written.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_link_sage import card  # noqa: E402

PRODUCTS = dict(num_nodes=2_449_029, num_edges=123_718_280, feat_dim=100, num_classes=47)
HIDDEN, FANOUTS, BATCH = 256, [25, 10], 1024


def device_ms(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    t1.synchronize()
    return t0.elapsed_time(t1) / reps


def composed_forward(tr):
    """The model's layer-wise forward through the pre-existing kernels (the A/B reference of the CSR mode)."""
    import torch
    from graphlearn_b200.ops import sage as S
    from graphlearn_b200.parallel.runtime import local_table_desc
    C, nodes, csr = tr.C, tr.nodes, tr.csr
    ip, idx = csr.indptr.local, csr.indices.local
    desc = nodes.feat_desc
    x_self = nodes.feats.local
    for l, c in enumerate(tr.convs):
        last = l == tr.L - 1
        d = c.in_self
        kp = S.pad_k(d)
        agg = C.gather_agg(desc, idx, ip, 0, 1 if c.agg_type == "mean" else 0)           # fp32 [n, d]
        a = torch.zeros(agg.size(0), 2 * kp, dtype=torch.bfloat16, device=agg.device)
        a[:, :d] = x_self[:agg.size(0), :d]
        a[:, kp:kp + d] = agg
        h = C.tc_linear_forward(a, tr.img[l], c.bias, tr.n_img[l], c.out_dim, not last, not last)
        if not last:
            desc, x_self = local_table_desc(h), h
    return h


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sampled-nodes", type=int, default=131072)
    ap.add_argument("--small", action="store_true", help="200k nodes / 10M edges (quick check)")
    args = ap.parse_args()
    import torch
    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.synthetic import make_sharded_graph
    rt = init()
    assert rt.is_cuda, "needs a CUDA device"
    shape = dict(PRODUCTS)
    if args.small:
        shape.update(num_nodes=200_000, num_edges=10_000_000)
    res = {"graph": dict(shape, feature_storage="bf16"), "model": "100-256-47 mean", "reps": args.reps}

    def trainer(skew):
        nodes, csr = make_sharded_graph(rt, feature_dtype=torch.bfloat16, seed=0, skew=skew, **shape)
        torch.manual_seed(0)
        model = EgoGraphSAGE(shape["feat_dim"], HIDDEN, shape["num_classes"], 2).to(rt.device)
        return FastSageTrainer(rt, nodes, csr, model, FANOUTS, BATCH, use_cuda_graph=False)

    for skew in (1.0, 0.0, 2.0):
        tr = trainer(skew)
        n, E = tr.nodes.n_local, tr.csr.n_edges
        ms = device_ms(tr.infer_all, args.reps)
        plan = tr._inf[0]
        rows = tr.L * (n + E)
        r = {"ms": round(ms, 3), "nodes_per_s": n / ms * 1e3, "gathered_rows": rows, "gathered_rows_per_s": rows / ms * 1e3,
             "gathered_GBps": (n + E) * (shape["feat_dim"] + HIDDEN) * 2 / ms / 1e6, "hub_rows": plan.n_hub,
             "hub_chunks": plan.n_chunks, "plan_deg": plan.plan_deg,
             "max_degree": int((tr.csr.indptr.local[1:] - tr.csr.indptr.local[:-1]).max())}
        if skew == 1.0:
            ref = composed_forward(tr)
            got = tr.infer_all()
            r["composed_ms"] = round(device_ms(lambda: composed_forward(tr), args.reps), 3)
            r["speedup_vs_composed"] = r["composed_ms"] / ms
            r["max_abs_diff_vs_composed"] = float((got - ref).abs().max())
            m = min(args.sampled_nodes, n) // BATCH * BATCH
            vids = torch.arange(m, device=rt.device)

            def sampled():
                for i in range(0, m, BATCH):
                    tr.predict(vids[i:i + BATCH])
            s_ms = device_ms(sampled, 1)
            r["sampled_predict"] = {"nodes": m, "ms": round(s_ms, 3), "nodes_per_s": m / s_ms * 1e3}
            r["speedup_vs_sampled_per_node"] = r["nodes_per_s"] / r["sampled_predict"]["nodes_per_s"]
        res["skew%g" % skew] = r
        del tr
        torch.cuda.empty_cache()
    res["skew2_vs_skew0_rows_per_s"] = res["skew2"]["gathered_rows_per_s"] / res["skew0"]["gathered_rows_per_s"]
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
