"""SPMD worker of tests/test_sage_inference_gpu.py::test_infer_all_two_ranks: ``infer_all`` on every rank (neighbour
rows of the hidden layer read from the peer's symmetric table) against the layer-wise forward of the all-gathered
graph computed on one device."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def main():
    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.ops import sage as S
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.synthetic import make_sharded_graph
    rt = init()
    W, r = rt.world, rt.rank
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=8)
    torch.manual_seed(0)
    tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2).to(rt.device), [10, 5], 128, use_cuda_graph=False)
    got = tr.infer_all()
    torch.cuda.synchronize()
    assert torch.equal(got, tr.infer_all())
    # the whole graph on every rank: features by vid, edges (src vid, dst vid)
    parts = rt.all_gather_object((nodes.feats.local[:, :100].float().cpu(), (csr._row_of_edge * W + r).cpu(),
                                  csr.indices.local.cpu()))
    n = sum(p[0].size(0) for p in parts)
    x = torch.zeros(n, 100)
    for q, p in enumerate(parts):
        x[q::W][:p[0].size(0)] = p[0]
    src = torch.cat([p[1] for p in parts])
    dst = torch.cat([p[2] for p in parts])
    dev = rt.device
    order = torch.argsort(src, stable=True)
    src, dst, h = src[order].to(dev), dst[order].to(dev), x.to(dev)
    deg = torch.bincount(src, minlength=n).double()
    for l, c in enumerate(tr.convs):
        last = l == len(tr.convs) - 1
        agg = torch.zeros(n, h.size(1), dtype=torch.float64, device=dev).index_add_(0, src, h.double()[dst])
        agg = (agg / deg.clamp(min=1)[:, None]).float()
        w = S.logical_weight(c.weight_p.detach(), c.in_self, c.in_nbr, c.agg_type).bfloat16().float()
        y = F.linear(torch.cat([h, agg], 1).bfloat16().float(), w, c.bias.detach())
        h = y if last else F.relu(y).bfloat16().float()
    ref = h[r::W][:nodes.n_local]
    err = float((got - ref).abs().max())
    assert err <= 2e-2 * float(ref.abs().max()), (err, float(ref.abs().max()))
    rt.barrier()
    if r == 0:
        print("DIST_INFER_OK")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
