"""The flagship path: hash-partitioned graph in HBM, fused sm_90a kernels, CUDA-graph step.
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 examples/train_sage_engine.py
(needs CUDA; on CPU use train_ego_sage.py)."""
import argparse

import torch

from common import sys  # noqa: F401  (fixes sys.path)

from graphlearn_b200.engine.fast_sage import FastSageTrainer
from graphlearn_b200.models.graphsage import EgoGraphSAGE
from graphlearn_b200.parallel.runtime import init
from graphlearn_b200.store.synthetic import make_sharded_graph
from graphlearn_b200.utils.checkpoint import save_checkpoint
from graphlearn_b200.utils.trace import ProgressLogger


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=2_449_029)
    ap.add_argument("--edges", type=int, default=123_718_280)
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--ckpt", default="")
    a = ap.parse_args(argv)
    rt = init()
    nodes, csr = make_sharded_graph(rt, a.nodes, a.edges, 100, 47)
    model = EgoGraphSAGE(100, 256, 47, 2).to(rt.device)
    tr = FastSageTrainer(rt, nodes, csr, model, [25, 10], 1024)
    gen = torch.Generator().manual_seed(rt.rank)
    seeds = lambda: torch.randint(0, nodes.n_local, (1024,), generator=gen) * rt.world + rt.rank  # noqa: E731
    tr.seeds.copy_(seeds().to(rt.device))
    tr.capture()
    prog = ProgressLogger(every=500)
    for it in range(a.steps):
        loss = tr.step(seeds())
        if (it + 1) % 500 == 0:
            torch.cuda.synchronize()
            if rt.rank == 0:
                print("step %d loss %.4f" % (it + 1, float(loss)))
        prog.update()
    if a.ckpt:
        save_checkpoint(a.ckpt, trainer=tr, rank=rt.rank)
    rt.shutdown()


if __name__ == "__main__":
    main()
