"""Sparse (edge_index) GCN node classification with train/val/test node masks, full 1-hop
neighbourhoods and data-parallel gradient averaging (graphlearn/examples/pytorch/gcn/train.py).
Runs on 1 GPU / CPU as is, or under torchrun on N GPUs (each rank trains on its own seeds).
   python examples/train_gcn_sparse.py"""
import argparse
import os
import tempfile

import numpy as np
import torch
import torch.nn.functional as F

from common import write_citation_like  # noqa: E402

import graphlearn_b200 as gl
from graphlearn_b200 import models
from graphlearn_b200.engine.loop import Trainer


def write_masks(d, n, seed=0):
    rs = np.random.RandomState(seed)
    perm = rs.permutation(n)
    out = {}
    for name, ids in (("train", perm[:int(0.6 * n)]), ("val", perm[int(0.6 * n):int(0.8 * n)]), ("test", perm[int(0.8 * n):])):
        p = os.path.join(d, name + "_table")
        with open(p, "w") as f:
            f.write("id:int64\tweight:float\n")
            for i in ids:
                f.write("%d\t1.0\n" % i)
        out[name] = p
    return out


def induce(res, device):
    """Star subgraphs (seed + all its neighbours, both edge directions) of one batch, concatenated into
    one edge_index with node offsets - the vectorised form of the reference's per-seed ``induce_func``."""
    src, nbr = res["src"], res["src_hop1"]
    xs = src.tensor("float_attrs")
    B = xs.size(0)
    counts = nbr.tensor("offsets") if "offsets" in nbr._t else torch.as_tensor(np.asarray(nbr.offsets), device=device)
    counts = counts.to(device).long()
    xn = nbr.tensor("float_attrs")
    x = torch.cat([xs, xn])
    seed_of_nbr = torch.repeat_interleave(torch.arange(B, device=device), counts)
    nbr_idx = B + torch.arange(xn.size(0), device=device)
    ei = torch.stack([torch.cat([seed_of_nbr, nbr_idx]), torch.cat([nbr_idx, seed_of_nbr])])
    return x, ei, src.tensor("labels").reshape(-1), B


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--epochs", type=int, default=4)
    ap.add_argument("--nodes", type=int, default=1500)
    ap.add_argument("--device", default=None)
    a = ap.parse_args(argv)
    d = tempfile.mkdtemp()
    node_f, edge_f, dim, classes = write_citation_like(d, n=a.nodes)
    masks = write_masks(d, a.nodes)
    gl.set_default_label(0)
    g = gl.Graph().node(node_f, "item", decoder=gl.Decoder(labeled=True, attr_types=["float"] * dim)) \
        .edge(edge_f, ("item", "item", "relation"), decoder=gl.Decoder(weighted=True), directed=False) \
        .node(masks["train"], "item", decoder=gl.Decoder(weighted=True), mask=gl.Mask.TRAIN) \
        .node(masks["val"], "item", decoder=gl.Decoder(weighted=True), mask=gl.Mask.VAL) \
        .node(masks["test"], "item", decoder=gl.Decoder(weighted=True), mask=gl.Mask.TEST) \
        .init(device=a.device)

    def query(mask, bs, shuffle):
        seed = g.V("item", mask=mask).batch(bs)
        seed = (seed.shuffle(traverse=True) if shuffle else seed).alias("src")
        seed.outV("relation").sample(0).by("full").alias("src_hop1")
        return gl.Dataset(seed.values())

    train_ds, test_ds = query(gl.Mask.TRAIN, 128, True), query(gl.Mask.TEST, 256, False)
    model = models.SparseGNN("gcn", dim, 32, classes, 2).to(g.device)

    def step(model, res):
        x, ei, y, B = induce(res, g.device)
        return F.cross_entropy(model(x, ei)[:B], y)

    def acc(model, res):
        x, ei, y, B = induce(res, g.device)
        return (model(x, ei)[:B].argmax(1) == y).float().mean()

    tr = Trainer(g.runtime, model, train_ds, step, lr=1e-2, log_every=10 ** 9)
    test_acc = 0.0
    for ep in range(a.epochs):
        loss = tr.train_epoch()
        test_acc = tr.evaluate(test_ds, acc)
        print("epoch %d loss %.4f test acc %.3f" % (ep, loss, test_acc))
    if g.runtime.world > 1:         # data-parallel replicas must hold identical parameters
        ps = g.runtime.all_gather_object(tr.flat_p.detach().cpu())
        assert all(torch.allclose(p, ps[0], atol=1e-6) for p in ps), "replicas diverged"
        print("replicas in sync on %d ranks" % g.runtime.world)
        # leave the process group before the interpreter exits: a rank that exits with it alive can abort in the
        # teardown of its gloo threads ("terminate called without an active exception")
        g.runtime.shutdown()
    return test_acc


if __name__ == "__main__":
    main()
