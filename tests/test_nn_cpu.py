"""CPU tests of the model layer, losses, feature encoding, checkpoint/resume and native loader."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import graphlearn_b200 as gl
from graphlearn_b200 import models
from graphlearn_b200 import nn as glnn
from tests import fixtures as fx


def test_ego_sage_conv_math():
    torch.manual_seed(0)
    for agg in ("mean", "sum", "gcn", "max"):
        c = glnn.EgoSAGEConv(6, 5, agg)
        x, nb = torch.randn(4, 6), torch.randn(12, 6)
        y = c(x, nb, 3)
        n3 = nb.view(4, 3, 6)
        if agg == "gcn":
            a = (x + n3.sum(1)) / 4
        else:
            a = torch.cat([x, {"mean": n3.mean(1), "sum": n3.sum(1), "max": n3.max(1).values}[agg]], 1)
        ref = F.linear(a, c.weight, c.bias)
        assert torch.allclose(y, ref, atol=1e-5), agg


def test_padded_weight_roundtrip():
    from graphlearn_b200.ops import sage as SG
    w = torch.randn(7, 100 + 100)
    wp = SG.pad_weight(w, 100, 100, "mean")
    assert wp.shape == (7, 256) and torch.equal(SG.logical_weight(wp, 100, 100, "mean"), w)
    assert float(wp[:, 100:128].abs().sum()) == 0 and float(wp[:, 228:].abs().sum()) == 0
    assert SG.fused_supported(100, 100, 256, "mean") and not SG.fused_supported(600, 600, 256, "mean")
    # unsplit headline layers (256 hidden, 47 classes over 256 + 256 padded inputs); 172 classes need 3 images of 64 columns
    assert SG.split_images(256, 256) == (1, 256) and SG.split_images(512, 47) == (1, SG.pad_n(47))
    assert SG.split_images(512, 172) == (3, 64) and SG.smem_fits(512, 64) and not SG.smem_fits(512, 96)
    # the Python fit check and the kernel's launch check size shared memory with the same formula
    from graphlearn_b200.parallel.runtime import native
    C = native()
    for k in (64, 128, 256, 512, 1024):
        for n in range(32, 257, 32):
            assert SG.smem_bytes(k, n) == C.sage_smem_bytes(k, n), (k, n)


def test_gat_softmax_rows_sum_to_one():
    s = torch.randn(10, 2)
    idx = torch.tensor([0, 0, 0, 1, 1, 2, 2, 2, 2, 3])
    a = glnn.segment_softmax(s, idx, 4)
    sums = torch.zeros(4, 2).index_add_(0, idx, a)
    assert torch.allclose(sums, torch.ones(4, 2), atol=1e-6)


def test_sparse_convs_vs_dense():
    torch.manual_seed(1)
    x = torch.randn(5, 4)
    ei = torch.tensor([[0, 0, 1, 2, 3, 4], [1, 2, 2, 3, 4, 0]])
    A = torch.zeros(5, 5)
    A[ei[0], ei[1]] = 1
    c = glnn.SAGEConv(4, 3, "mean")
    ref = c.lin_self(x) + c.lin_nbr((A @ x) / A.sum(1, keepdim=True).clamp(min=1))
    assert torch.allclose(c(x, ei), ref, atol=1e-5)
    g = glnn.GCNConv(4, 3)
    Ah = A + torch.eye(5)
    d = Ah.sum(1).pow(-0.5)
    ref = (d[:, None] * Ah * d[None, :]) @ g.lin(x) + g.bias
    assert torch.allclose(g(x, ei), ref, atol=1e-5)


def test_losses():
    L = glnn.loss
    pos, neg = torch.tensor([10.0, 10.0]), torch.tensor([-10.0, -10.0, -10.0])
    assert float(L.sigmoid_cross_entropy_loss(pos, neg)) < 1e-3
    s = torch.eye(3)
    l = L.unsupervised_softmax_cross_entropy_loss(s * 10, s * 10, -s.repeat_interleave(2, 0) * 10)
    assert float(l) < 1e-3
    z = torch.zeros(2, 3)
    assert float(L.triplet_margin_loss(z, z, z, z, z, z, margin=1.0)) == pytest.approx(1.0)
    assert float(L.triplet_softplus_loss(z, z, z, z, z, z)) == pytest.approx(2 * np.log(2), abs=1e-5)


def test_feature_encoder_fused_tables():
    d = gl.Decoder(attr_types=["float", ("int", 10), ("string", 20), ("int", 5), "int", "float"],
                   attr_dims=[None, 8, 8, 4, None, None])
    spec = d.feature_spec
    enc = glnn.FeatureEncoder(spec)
    assert set(enc.tables.keys()) == {"8", "4"}           # two dim-8 columns fused into one table
    assert enc.tables["8"].num_embeddings == 30
    out = enc(torch.randn(6, 2), torch.randint(0, 100, (6, 4)))
    assert out.shape == (6, enc.output_dim) and enc.output_dim == 2 + 1 + 8 + 8 + 4


def test_node2vec_pairs_and_model():
    path = torch.arange(12).view(2, 6)
    s, d = models.gen_pair(path, 1, 1)
    assert s.numel() == 2 * (6 * 2 - 2)
    m = models.Node2Vec(50, 8, sparse=False)
    loss = m(torch.tensor([1, 2]), torch.tensor([3, 4]), torch.randint(0, 50, (2, 5)))
    loss.backward()
    assert m.src_emb.weight.grad is not None


def test_seal_labels_and_model():
    ds = torch.tensor([0, 1, 1, 2, 2 ** 31 - 1])
    dd = torch.tensor([1, 0, 1, 1, 2])
    z = models.drnl_node_labeling(ds, dd)
    assert z[0] == 1 and z[1] == 1 and z[4] == 0 and z[2] == 2
    m = models.SEAL(4, 8, num_layers=2)
    ei = torch.tensor([[0, 1, 2, 3], [2, 2, 3, 0]])
    out = m(torch.randn(5, 4), ei, z)
    assert out.shape == ()


def test_ego_gnn_variants_and_bipartite():
    xs = [torch.randn(4, 6), torch.randn(12, 6), torch.randn(24, 6)]
    for kind in ("sage", "gat", "gin"):
        m = models.make_ego_gnn(kind, 6, 8, 3, 2)
        assert m(xs, [3, 2]).shape == (4, 3)
    b = models.EgoBipartiteSAGE(6, 5, 8, 4, hops=2)
    u = [torch.randn(4, 6), torch.randn(8, 5), torch.randn(16, 6)]
    i = [torch.randn(4, 5), torch.randn(8, 6), torch.randn(16, 5)]
    ue, ie = b(u, i, [2, 2], [2, 2])
    assert ue.shape == (4, 4) and ie.shape == (4, 4)
    assert float(b.in_batch_negative_loss(ue, ie)) > 0


def test_nn_dataset_egograph(tmp_path):
    g = fx.build_graph(fx.write_graph(str(tmp_path)))
    q = g.V("item").batch(5).alias("s").outV("sim").sample(2).by("topk").alias("h1") \
         .outV("sim").sample(2).by("topk").alias("h2").values()
    ds = glnn.Dataset(q)
    ego = ds.get_egograph("s", ["h1", "h2"])
    assert ego.nbr_nums == [2, 2]
    assert ego.src.floats.shape == (5, 4) and ego.hop_node(1).floats.shape == (20, 4)
    m = models.EgoGraphSAGE(4, 8, 3, 2, bf16_activations=False)
    out = m([h.floats for h in ego.hops()], ego.nbr_nums)
    assert out.shape == (5, 3)
    # neighbors=None: the hop chain is read off the query (single positive downstream per hop); edge hops are skipped
    auto = glnn.Dataset(q).get_egograph("s")
    assert auto.nbr_nums == [2, 2] and auto.hop_node(1).floats.shape == (20, 4)
    src = g.V("item").batch(5).alias("r")
    src.outE("sim").sample(2).by("topk").alias("e1").inV().alias("n1")
    assert glnn.Dataset(src.values()).get_egograph("r").nbr_nums == [2]
    fork = g.V("item").batch(5).alias("f")
    fork.outV("sim").sample(2).by("topk").alias("a")
    fork.outV("sim").sample(3).by("random").alias("b")
    with pytest.raises(ValueError):
        glnn.Dataset(fork.values()).get_egograph("f")


def test_checkpoint_resume_is_deterministic(tmp_path):
    """model + optimizer + RNG + traversal state round-trip: resumed run == uninterrupted run."""
    from graphlearn_b200.engine.trainer import SageTrainer
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.synthetic import make_sharded_graph
    from graphlearn_b200.utils.checkpoint import load_checkpoint, save_checkpoint
    rt = init(device="cpu")
    nodes, csr = make_sharded_graph(rt, 500, 4000, 16, 4, seed=2)

    def mk():
        torch.manual_seed(0)
        return SageTrainer(rt, nodes, csr, models.EgoGraphSAGE(16, 8, 4, 2), [3, 2], 32, lr=1e-2, seed=5)

    seeds = [torch.randint(0, 500, (32,), generator=torch.Generator().manual_seed(i)) for i in range(8)]
    a = mk()
    la = [float(a.step(s)) for s in seeds]
    b = mk()
    for s in seeds[:4]:
        b.step(s)
    save_checkpoint(str(tmp_path / "ck"), trainer=b)
    c = mk()
    load_checkpoint(str(tmp_path / "ck"), trainer=c)
    lc = [float(c.step(s)) for s in seeds[4:]]
    assert np.allclose(lc, la[4:], rtol=1e-5, atol=1e-6), (lc, la[4:])


def test_embedding_dump_roundtrip(tmp_path):
    from graphlearn_b200.utils.checkpoint import embedding_decoder, save_embeddings
    ids = torch.arange(10) * 3
    emb = torch.randn(10, 6)
    p = str(tmp_path / "emb.txt")
    save_embeddings(p, ids, emb)
    assert open(p).readline().strip() == "id:int64\temb:string"
    g = gl.Graph().node(p, "e", decoder=embedding_decoder(6)).init(device="cpu")
    back = g.lookup_nodes("e", ids.numpy()).float_attrs
    assert np.allclose(back, emb.numpy(), atol=1e-4)


def test_loader_rejects_malformed(tmp_path):
    p = tmp_path / "bad.tsv"
    p.write_text("id:int64\tfeature:string\n1\t0.5:xx\n")
    g = gl.Graph().node(str(p), "n", decoder=gl.Decoder(attr_types=["float", "float"]))
    with pytest.raises(RuntimeError):
        g.init(device="cpu")


def test_config_setters_and_errors():
    gl.set_default_neighbor_id(-3)
    gl.set_padding_mode(gl.REPLICATE)
    gl.set_inner_threadnum(7)
    cfg = gl.get_config()
    assert cfg.default_neighbor_id == -3 and cfg.padding_mode == gl.REPLICATE and cfg.inter_threadnum == 7
    assert issubclass(gl.OutOfRangeError, gl.errors.GLError) and gl.OutOfRangeError().error_code == 11
    assert gl.errors.exception_type_from_error_code(5) is gl.errors.NotFoundError
    assert gl.strategy2op("edge_weight") == "EdgeWeightSampler"
    assert gl.get_mask_type("i", gl.Mask.TRAIN) == "MASKTRAIN_i"


def test_generic_trainer_loop(tmp_path):
    """engine.loop.Trainer over a GSL dataset: loss decreases, epoch ends on OutOfRange, ckpt written."""
    from graphlearn_b200.engine.loop import Trainer
    g = fx.build_graph(fx.write_graph(str(tmp_path / "g")))
    q = g.V("user").batch(8).shuffle(traverse=True).alias("u").outV("buy").sample(3).by("edge_weight").alias("i").values()
    ds = gl.Dataset(q)
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(4, 16), torch.nn.ReLU(), torch.nn.Linear(16, 3))

    def step(m, b):
        x = b["i"].tensor("float_attrs").mean(1)
        return F.cross_entropy(m(x), b["u"].tensor("labels"))

    tr = Trainer(g.runtime, model, ds, step, lr=2e-2, ckpt_path=str(tmp_path / "ck"), ckpt_every=5, log_every=1000)
    first = tr.train_epoch()
    for _ in range(15):
        last = tr.train_epoch()
    assert tr.global_step == 16 * (fx.N_USER // 8) and last < first
    assert os.path.exists(str(tmp_path / "ck") + ".rank0")


def test_sharded_embedding_sparse_sgd():
    from graphlearn_b200.parallel.runtime import init
    rt = init(device="cpu")
    emb = glnn.ShardedEmbedding(rt, 50, 8, lr=0.5)
    w0 = emb.local_weight().clone()
    ids = torch.tensor([[1, 2], [2, 7]])
    out = emb(ids)
    assert out.shape == (2, 2, 8) and torch.allclose(out[0, 0], w0[1])
    out.sum().backward()
    w1 = emb.local_weight()
    assert torch.allclose(w1[1], w0[1] - 0.5) and torch.allclose(w1[2], w0[2] - 1.0) and torch.allclose(w1[3], w0[3])



def test_sharded_embedding_sparse_adam_cpu():
    """portable path of the sparse Adam update (touched rows only, duplicates summed, global-step bias correction)"""
    import torch
    from graphlearn_b200 import nn as glnn
    from graphlearn_b200.parallel.runtime import init
    rt = init(device="cpu")
    emb = glnn.ShardedEmbedding(rt, 50, 8, lr=0.01, optimizer="adam")
    w = emb.local_weight().clone().double()
    m, v = torch.zeros_like(w), torch.zeros_like(w)
    g = torch.Generator().manual_seed(1)
    for t in range(1, 6):
        ids = torch.randint(0, 50, (16,), generator=g)
        grad = torch.randn(16, 8, generator=g)
        emb(ids).backward(grad)
        uniq, inv = torch.unique(ids, return_inverse=True)
        gs = torch.zeros(uniq.numel(), 8, dtype=torch.float64).index_add_(0, inv, grad.double())
        m[uniq] = 0.9 * m[uniq] + 0.1 * gs
        v[uniq] = 0.999 * v[uniq] + 0.001 * gs * gs
        w[uniq] -= 0.01 / (1 - 0.9 ** t) * m[uniq] / (v[uniq].sqrt() / (1 - 0.999 ** t) ** 0.5 + 1e-8)
    assert torch.allclose(emb.local_weight(), w.float(), rtol=1e-4, atol=1e-6)


def test_pyg_style_loader_and_cluster_helpers(tmp_path):
    """P8: TorchDataset + induce_func -> list of subgraphs -> PyGDataLoader -> collated Batch."""
    import graphlearn_b200 as gl
    from graphlearn_b200 import nn as glnn
    from graphlearn_b200.cluster import get_cluster_spec, launch_server
    from tests import fixtures as fx
    d = fx.write_graph(str(tmp_path))
    g = gl.Graph().node(d + "/item.tsv", "item", decoder=gl.Decoder(attr_types=["float"] * 4)) \
        .edge(d + "/i2i.tsv", ("item", "item", "sim"), decoder=gl.Decoder(labeled=True, timestamped=True))
    launch_server(g)                                   # == init()
    assert get_cluster_spec(world_size=2)["client_count"] == 2
    q = g.V("item").batch(5).alias("src").outV("sim").sample(3).by("random").alias("n1").values()

    def induce(data):
        src, n1 = data["src"], data["n1"]
        out = []
        for i in range(src.ids.numel()):
            x = torch.cat([src.floats[i:i + 1], n1.floats[3 * i:3 * i + 3]])
            ei = torch.tensor([[0, 0, 0], [1, 2, 3]], device=x.device)
            out.append(glnn.SubGraphData(x, ei, y=src.ids[i:i + 1]))
        return out
    loader = glnn.PyGDataLoader(glnn.TorchDataset(q, transform=induce), length=3)
    batches = list(loader)
    assert len(batches) == 3
    b = batches[0]
    assert b.num_graphs == 5 and b.x.shape == (20, 4) and b.edge_index.shape == (2, 15)
    assert b.edge_index[:, 3:6].tolist() == [[4, 4, 4], [5, 6, 7]] and b.batch.tolist() == sum([[i] * 4 for i in range(5)], [])


def test_relabel_and_spmm_portable():
    from graphlearn_b200.ops.sparse import Relabel, spmm
    ids = torch.tensor([[7, 3, 7], [-1, 9, 3]])
    r = Relabel(ids)
    assert r.uniq.tolist() == [7, 3, 9] and r.inverse.tolist() == [[0, 1, 0], [-1, 2, 1]]
    assert r.lookup(torch.tensor([9, 4, 7, -1])).tolist() == [2, -1, 0, -1]
    x = torch.randn(5, 6, requires_grad=True)
    row, col = torch.tensor([0, 0, 2, 4]), torch.tensor([1, 3, 3, 0])
    w = torch.rand(4, 2, requires_grad=True)
    out = spmm(x, row, col, w, 5, heads=2)
    ref = torch.zeros(5, 2, 3).index_add_(0, row, x[col].view(-1, 2, 3) * w[:, :, None]).reshape(5, 6)
    assert torch.allclose(out, ref)


def test_hetero_conv_and_link_predictor():
    """HeteroConv: per-edge-type convs, results for the same destination type are aggregated; bipartite convs get
    [x_src, x_dst]; LinkPredictor returns one logit per pair."""
    from graphlearn_b200 import nn as glnn
    torch.manual_seed(0)
    xu, xi = torch.randn(5, 6), torch.randn(7, 4)
    ei_ui = torch.tensor([[0, 1, 1, 6], [0, 0, 4, 2]])          # rows: items, cols: users
    ei_ii = torch.tensor([[0, 1, 2, 3], [1, 2, 3, 0]])
    conv = glnn.HeteroConv({("u", "buy", "i"): glnn.BipartiteSAGEConv(6, 4, 8),
                            ("i", "sim", "i"): glnn.SAGEConv(4, 8)}, agg_type="sum")
    out = conv({("u", "buy", "i"): ei_ui, ("i", "sim", "i"): ei_ii}, {"u": xu, "i": xi})
    assert set(out) == {"i"} and out["i"].shape == (7, 8)
    a = conv.convs[0](ei_ui, [xu, xi])
    b = conv.convs[1](ei_ii, xi)
    assert torch.allclose(out["i"], a + b, atol=1e-6)
    # closed form of the bipartite conv for item 1: mean of users 0 and 4
    c0 = conv.convs[0]
    want = c0.lin_self(xi[1]) + c0.lin_nbr((xu[0] + xu[4]) / 2)
    assert torch.allclose(a[1], want, atol=1e-5)
    lp = glnn.LinkPredictor(8, num_layers=2)
    assert lp(torch.randn(9, 8)).shape == (9,)
    sg = glnn.HeteroSubGraph({("u", "buy", "i"): ei_ui}, {"u": glnn.Data(ids=torch.arange(5)), "i": glnn.Data(ids=torch.arange(7))})
    assert sg.num_nodes("i") == 7 and sg.num_edges(("u", "buy", "i")) == 4 and sg.edge_types == [("u", "buy", "i")]


def test_temporal_graph_container(tmp_path):
    """nn.Dataset.get_temporalgraph: centre times, per-hop edge times, time spans >= 0 under the temporal filter."""
    import os
    import graphlearn_b200 as gl
    from graphlearn_b200 import nn as glnn
    d = str(tmp_path)
    with open(d + "/n.tsv", "w") as f:
        f.write("id:int64\ttimestamp:int64\tfeature:string\n" + "".join("%d\t%d\t%d:%d\n" % (i, 100 + 10 * i, i, i) for i in range(20)))
    with open(d + "/e.tsv", "w") as f:
        f.write("src_id:int64\tdst_id:int64\ttimestamp:int64\n")
        for i in range(20):
            for k in range(1, 4):
                f.write("%d\t%d\t%d\n" % (i, (i + k) % 20, 95 + 10 * i - k))
    gl.set_default_neighbor_id(-1)
    gl.set_padding_mode(gl.REPLICATE)
    g = gl.Graph().node(d + "/n.tsv", "n", decoder=gl.Decoder(timestamped=True, attr_types=["float", "float"])) \
        .edge(d + "/e.tsv", ("n", "n", "e"), decoder=gl.Decoder(timestamped=True)).init(device="cpu")
    src = g.V("n").batch(5).alias("s")
    src.outE("e").sample(2).by("topk").alias("e1").inV().alias("h1")
    ds = glnn.Dataset(src.values())
    tg = ds.get_temporalgraph("s", ["e1"], ["h1"])
    assert tg.nbr_nums == [2] and tg.src_t.tolist() == [100, 110, 120, 130, 140]
    spans = tg.time_spans()[0].reshape(5, 2)
    assert (spans == torch.tensor([[6, 7]] * 5)).all()          # edge times 95+10i-k, most recent first: k = 1, 2
    enc = tg.transform(glnn.TimeEncoder(8))
    assert enc.nbr_t[0].shape == (10, 8) and enc.src_t.shape == (5, 8)


def test_step_profiler_writes_chrome_traces(tmp_path):
    import json
    from graphlearn_b200.utils.trace import DeviceTimer, StepProfiler
    prof = StepProfiler(str(tmp_path), start=2, stop=7, every=2)
    x = torch.randn(64, 64)
    timer = DeviceTimer()
    for step in range(8):
        with prof.step(step), timer.section("mm"):
            (x @ x).sum().item()
    assert [os.path.basename(p) for p in prof.written] == ["timeline_2.json", "timeline_4.json", "timeline_6.json"]
    assert "traceEvents" in json.load(open(prof.written[0]))
    assert timer.summary()["mm"]["calls"] == 8


def test_multival_token_hash_is_process_independent():
    """string tokens must land in the same embedding bucket in every process (ranks, train vs serve)."""
    import subprocess
    import sys
    from graphlearn_b200.nn.feature import _hash_token
    code = "import sys; sys.path.insert(0, %r); from graphlearn_b200.nn.feature import _hash_token; print(_hash_token('brand_42'), _hash_token(''))" % \
        os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = {subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, PYTHONHASHSEED=str(s))).stdout.strip()
            for s in (1, 2)}
    assert outs == {"%d %d" % (_hash_token("brand_42"), _hash_token(""))}


def test_stall_detector_fires_once_and_rearms():
    import time
    from graphlearn_b200.utils.watchdog import StallDetector
    hits = []
    sd = StallDetector(timeout_s=0.6, on_stall=lambda idle: hits.append(idle), poll_s=0.05).start()
    for _ in range(5):                       # a healthy loop never trips it
        time.sleep(0.05); sd.tick()
    assert hits == []
    time.sleep(1.5)                          # a hang does, exactly once
    assert len(hits) == 1 and hits[0] > 0.6
    sd.tick(); time.sleep(1.5)               # re-armed by the next step
    assert len(hits) == 2
    sd.stop()


def test_feature_columns_groups_and_handler():
    """nn/feature_column.py (feature_column.py / feature_handler.py of the reference): every column kind, the spec-driven
    grouping (per-feature, fused by width, dynamic, multi-value strings) and the concatenation order."""
    torch.manual_seed(0)
    num = glnn.NumericColumn("x", normalizer_func=lambda v: v / 10)
    assert num(torch.tensor([10, 20])).tolist() == [1.0, 2.0]
    emb = glnn.EmbeddingColumn("e", 7, 3)
    assert torch.equal(emb(torch.tensor([2, 99])), emb.table.weight[[2, 6]])              # out-of-range ids clamp
    hashed = glnn.EmbeddingColumn("h", 7, 3, need_hash=True)
    assert hashed(torch.tensor([123456789, 5])).shape == (2, 3)
    fused = glnn.FusedEmbeddingColumn("f", [4, 6], 2)
    out = fused([torch.tensor([1, 3]), torch.tensor([0, 5])])
    assert out.shape == (2, 4) and torch.equal(out[1], torch.cat([fused.table.weight[3], fused.table.weight[4 + 5]]))
    sp = glnn.SparseEmbeddingColumn("s", 50, 4, delimiter=",")
    o = sp(np.array(["a,b", "", "b"], dtype=object))
    assert torch.allclose(o[1], torch.zeros(4)) and not torch.allclose(o[2], torch.zeros(4))
    assert torch.allclose(o[0] - o[2], sp(np.array(["a"], dtype=object))[0], atol=1e-6)
    dyn = glnn.DynamicEmbeddingColumn("d", 3, is_string=True)
    a = dyn(["tok1", "tok2", "tok1"])
    assert torch.equal(a[0], a[2]) and dyn.table.num_keys == 2
    dyn.eval()
    assert torch.allclose(dyn(["never seen"]), torch.zeros(1, 3)) and dyn.table.num_keys == 2
    dsp = glnn.DynamicSparseEmbeddingColumn("ds", 2, delimiter="|")
    assert dsp(["x|y", "y"]).shape == (2, 2) and dsp.table.num_keys == 2
    grp = glnn.FeatureGroup([glnn.NumericColumn("a"), glnn.EmbeddingColumn("b", 5, 2)])
    assert grp([torch.tensor([1.0, 2.0]), torch.tensor([0, 4])]).shape == (2, 3) and len(grp) == 2
    with pytest.raises(ValueError):
        grp([torch.tensor([1.0])])

    spec = gl.FeatureSpec(8)
    spec.append_dense()                       # float 0
    spec.append_dense()                       # float 1
    spec.append_dense(is_float=False)         # int 0: integer treated like a float
    spec.append_sparse(10, 4, False)          # int 1: fused (width 4)
    spec.append_sparse(20, 4, False)          # int 2: fused (width 4)
    spec.append_sparse(30, 3, True)           # int 3: hashed, own table
    spec.append_sparse(None, 5, True)         # int 4: dynamic vocabulary of hashed keys
    spec.append_multival(40, 2, ":")          # string 0
    spec.append_multival(None, 6, ":")        # string 1: dynamic multi-value
    assert spec.dimension == 1 + 1 + 1 + 4 + 4 + 3 + 5 + 2 + 6
    assert isinstance(spec.int_specs[4], gl.DynamicSparseSpec) and isinstance(spec.string_specs[1], gl.DynamicMultivalSpec)
    fh = glnn.FeatureHandler("item", spec)
    assert fh.output_dim == spec.dimension
    n = 6
    data = glnn.Data(ids=torch.arange(n), floats=torch.rand(n, 2),
                     ints=torch.stack([torch.arange(n), torch.arange(n) % 10, torch.arange(n) % 20, torch.arange(n) * 7919,
                                       torch.arange(n) * 104729], 1),
                     strings=np.array([["a:b", "p:q:r"]] * n, dtype=object))
    y = fh(data)
    assert y.shape == (n, spec.dimension)
    assert torch.allclose(y[:, :2], data.floats) and torch.allclose(y[:, 2], torch.arange(n).float())     # floats, then dense int
    # order after the per-feature int columns [dense(1) | hashed(3) | dynamic(5)]: the fused group, then the strings
    fcol = fh._fused_int_fg[0]
    want = torch.cat([fcol.table.weight[data.ints[:, 1]], fcol.table.weight[10 + data.ints[:, 2]]], 1)
    assert torch.allclose(y[:, 2 + 1 + 3 + 5:2 + 1 + 3 + 5 + 8], want)
    y.sum().backward()
    assert fcol.table.weight.grad is not None and fh._string_fg[1].table.weight.grad is not None
    # without fusing every sparse column owns its table
    assert len(glnn.FeatureHandler("x", spec, fuse_embedding=False)._fused_int_fg) == 0


def test_reference_named_models_base_classes_and_torch_utils(tmp_path):
    """Names a reference user expects: nn.Module / EgoConv / SubConv / LinearLayer, models.GCN / GraphSAGE / GAT over a
    BatchGraph, unsorted_segment_softmax, the nn.pytorch data utils and the end-of-training barrier hook."""
    from graphlearn_b200.nn import utils as U
    assert issubclass(glnn.EgoSAGEConv, glnn.Module) and glnn.unsorted_segment_softmax is glnn.segment_softmax

    class MyConv(glnn.EgoConv):
        def forward(self, x, neighbor, expand):
            return x + neighbor.reshape(x.size(0), expand, -1).mean(1)
    layer = glnn.EgoLayer([MyConv()])
    out = layer([torch.ones(2, 3), torch.ones(8, 3)], [4])
    assert torch.allclose(out[0], torch.full((2, 3), 2.0))
    with pytest.raises(NotImplementedError):
        glnn.SubConv()(None, None)
    lin = glnn.LinearLayer("l", 3, 5, activation=torch.relu)
    assert lin(torch.randn(4, 3)).shape == (4, 5) and glnn.LinearLayer("lazy", None, 2)(torch.randn(4, 7)).shape == (4, 2)
    # a BatchGraph of 3 path graphs with 4 nodes each
    ei = torch.cat([torch.tensor([[0, 1, 2], [1, 2, 3]]) + 4 * i for i in range(3)], 1)
    bg = glnn.BatchGraph(ei, glnn.Data(ids=torch.arange(12), floats=torch.randn(12, 6)), graph_node_offsets=torch.tensor([0, 4, 8, 12]))
    for cls, kw in ((models.GCN, {}), (models.GraphSAGE, {"agg_type": "sum"}), (models.GAT, {"attn_heads": 2})):
        m = cls(3, 6, 8, 5, depth=2, drop_rate=0.1, **kw)
        src, dst = m(bg)
        assert src.shape == (3, 5) and dst.shape == (3, 5)
        (src * dst).sum().backward()
    assert bg.transform().nodes.shape == (12, 6) and bg.transform().num_nodes == 12
    # process-level helpers
    U._reset_for_tests()
    assert U.get_world_size() == 1 and U.get_rank() == 0 and U.get_num_client() == 1
    U._reset_for_tests()
    U.set_client_num(3)
    assert U.get_num_client() == 3
    spec = U.get_cluster_spec()
    host, port = spec["server"].split(":")
    assert int(port) > 0 and spec["client_count"] == 3 and not U.is_server_launched()
    hook = glnn.SyncBarrierHook()
    with hook:
        pass                                            # no process group: returns at once
    hook.end()
    U._reset_for_tests()
    # Collater / worker_init_fn
    items = [glnn.SubGraphData(torch.ones(2, 3), torch.tensor([[0], [1]])), glnn.SubGraphData(torch.ones(3, 3), torch.tensor([[0, 1], [1, 2]]))]
    b = glnn.Collater()([items])
    assert b.num_graphs == 2 and b.x.shape == (5, 3) and b.edge_index.tolist() == [[0, 2, 3], [1, 3, 4]]
    assert glnn.Collater()([torch.ones(2), torch.zeros(2)]).shape == (2, 2)
    glnn.worker_init_fn(0)                              # outside a worker: no-op


def test_temporal_dataset_and_loader(tmp_path):
    """nn.TemporalDataset / TemporalDataLoader (nn/pytorch/data/temporal_dataset.py): an edge-rooted query streams
    TemporalData(src, dst, t, msg) batches for one epoch."""
    d = str(tmp_path)
    with open(d + "/n.tsv", "w") as f:
        f.write("id:int64\tfeature:string\n" + "".join("%d\t%d\n" % (i, i) for i in range(10)))
    with open(d + "/e.tsv", "w") as f:
        f.write("src_id:int64\tdst_id:int64\tweight:float\ttimestamp:int64\n")
        for i in range(23):
            f.write("%d\t%d\t%.1f\t%d\n" % (i % 10, (i * 3) % 10, 0.5 * i, 1000 + i))
    g = gl.Graph().node(d + "/n.tsv", "n", decoder=gl.Decoder(attr_types=["float"])) \
        .edge(d + "/e.tsv", ("n", "n", "e"), decoder=gl.Decoder(weighted=True, timestamped=True)).init(device="cpu")
    q = g.E("e").batch(8).alias("event").values()
    loader = glnn.TemporalDataLoader(glnn.TemporalDataset(q, event_name="event"), batch_size=99, shuffle=True)
    batches = list(loader)
    assert [b.num_events for b in batches] == [8, 8, 7]
    t = torch.cat([b.t for b in batches])
    assert sorted(t.tolist()) == list(range(1000, 1023))
    b0 = batches[0]
    assert torch.equal(b0.dst, (3 * (b0.t - 1000)) % 10) and torch.allclose(b0.msg.reshape(-1), 0.5 * (b0.t - 1000).float())
    with pytest.raises(ValueError):
        next(iter(glnn.TemporalDataset(g.E("e").batch(4).alias("x").values(), event_name="event")))
    g.close()


def test_eval_metrics_recall_ndcg_f1():
    """utils/metrics.py (examples/eval of the reference): hand-checked Recall / NDCG / HitRate, the vectorised form agrees,
    KNN-recall evaluation through Graph.search, multi-label F1 on separable embeddings."""
    from graphlearn_b200.utils import metrics as M
    gt = [[1, 2, 3], [9], [5, 6]]
    rec = np.array([[2, 7, 1, 8], [4, 5, 6, 7], [6, 5, 0, 1]])
    r, n, h = M.eval_metrics(gt, rec)
    dcg0 = 1 / np.log2(2) + 1 / np.log2(4)
    idcg0 = 1 / np.log2(2) + 1 / np.log2(3)
    assert abs(r - (2 / 3 + 0 + 1.0)) < 1e-9 and h == 2 and abs(n - (dcg0 / idcg0 + 1.0)) < 1e-9
    v = M.recall_metrics_at_k(torch.from_numpy(rec), torch.tensor([[1, 2, 3], [9, -1, -1], [5, 6, -1]]))
    assert abs(v["recall"] - r / 3) < 1e-9 and abs(v["ndcg"] - n / 3) < 1e-9 and abs(v["hit_rate"] - 2 / 3) < 1e-9
    # KNN recall: items on a circle, a user's ground truth = the 3 items nearest to its embedding
    ang = np.linspace(0, 2 * np.pi, 40, endpoint=False)
    items = np.stack([np.cos(ang), np.sin(ang)], 1).astype(np.float32)
    users = items[[3, 17, 30]] * 0.9
    g = gl.Graph().node({"ids": np.arange(40), "float_attrs": items}, "i", decoder=gl.Decoder(attr_types=["float"] * 2))
    g.edge({"src_ids": np.arange(40), "dst_ids": (np.arange(40) + 1) % 40}, ("i", "i", "e")).init(device="cpu")
    res = M.evaluate_recall(g, "i", users, [[2, 3, 4], [16, 17, 18], [29, 30, 31]], top_k=3)
    assert res["recall"] == 1.0 and res["hit_rate"] == 1.0 and res["ndcg"] == 1.0
    g.close()
    rs = np.random.RandomState(0)
    lab = rs.rand(300, 4) < 0.4
    lab[:, 0] |= ~lab.any(1)
    emb = lab.astype(np.float64) + 0.05 * rs.randn(300, 4)
    f1 = M.multilabel_f1(emb, lab, train_ratios=(0.5,), shuffles=1)
    assert f1[0.5]["micro"] > 0.95 and f1[0.5]["macro"] > 0.95


def test_local_and_dist_trainer_reference_surface(tmp_path):
    """engine/trainers.py: LocalTrainer / DistTrainer with the reference trainers' method names - train (periodic checkpoints,
    resume), test, train_and_evaluate, save_node_embedding(_bigdata), join."""
    from graphlearn_b200.engine.trainers import DistTrainer, LocalTrainer
    g = fx.build_graph(fx.write_graph(str(tmp_path / "g")))

    def make_ds():
        return gl.Dataset(g.V("user").batch(8).shuffle(traverse=True).alias("u").outV("buy").sample(3).by("edge_weight").alias("i").values())

    def step(m, b):
        return F.cross_entropy(m(b["i"].tensor("float_attrs").mean(1)), b["u"].tensor("labels"))

    def acc(m, b):
        return (m(b["i"].tensor("float_attrs").mean(1)).argmax(1) == b["u"].tensor("labels")).float().mean()

    def embed(m, b):
        return b["u"].ids_t, m(b["i"].tensor("float_attrs").mean(1))
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Linear(4, 16), torch.nn.ReLU(), torch.nn.Linear(16, 3))
    ck = str(tmp_path / "ckpt")
    tr = LocalTrainer(ckpt_dir=ck, save_checkpoint_secs=None, save_checkpoint_steps=4, progress_steps=1000)
    first = tr.train(make_ds(), model, step, learning_rate=2e-2, epochs=1)
    loss, metric = tr.train_and_evaluate(make_ds(), make_ds(), model, step, acc, learning_rate=2e-2, epochs=10)
    assert loss < first and 0.0 <= metric <= 1.0
    steps_per_epoch = fx.N_USER // 8
    assert tr.global_step == 11 * steps_per_epoch                 # the second call resumed from the first one's checkpoint
    assert os.path.exists(os.path.join(ck, "model.ckpt.rank0"))
    # a fresh trainer + fresh model pick the checkpoint up (parameters and step counter)
    model2 = torch.nn.Sequential(torch.nn.Linear(4, 16), torch.nn.ReLU(), torch.nn.Linear(16, 3))
    tr2 = LocalTrainer(ckpt_dir=ck, save_checkpoint_secs=0.0001, progress_steps=1000)        # time-based checkpoints: step-wise loop
    tr2.train(make_ds(), model2, step, learning_rate=2e-2, epochs=1)
    assert tr2.global_step == 12 * steps_per_epoch
    assert abs(tr2.test(make_ds(), model2, acc) - tr.test(make_ds(), model, acc)) < 0.35
    out = str(tmp_path / "emb.txt")
    tr2.save_node_embedding(out, make_ds(), model2, embed)
    lines = open(out + ".rank0").read().strip().split("\n")
    assert lines[0] == "id:int64\temb:string" and len(lines) == 1 + fx.N_USER
    tr2.save_node_embedding_bigdata(str(tmp_path / "big.txt"), make_ds(), model2, embed, block_max_lines=20)
    assert len([f for f in os.listdir(str(tmp_path)) if f.startswith("big")]) == (fx.N_USER + 19) // 20
    dt = DistTrainer(cluster_spec={"worker": ["a"]}, job_name="worker", ckpt_dir=None, progress_steps=1000)
    assert dt.is_chief and dt.worker_count == 1 and not dt.is_local
    dt.train(make_ds(), model, step, learning_rate=1e-2, epochs=1)
    dt.join()


def test_link_dist_trainer_hits_and_predict(tmp_path):
    """engine/trainers.LinkDistTrainer (examples/tf/link_trainer.py): dot-product link model on the user-item fixture - trained
    on positive edges + sampled negatives, Hits@K on held-out positive / negative streams rises above the untrained model,
    predict writes scored edges; hits_at_k matches its definition on a hand example."""
    from graphlearn_b200.engine.trainers import LinkDistTrainer
    from graphlearn_b200.utils.metrics import hits_at_k
    assert hits_at_k([0.9, 0.2, 0.5], [0.1, 0.3, 0.6, 0.4], 2) == pytest.approx(2 / 3)      # 2nd best negative = 0.4
    assert hits_at_k([0.9], [0.1], 5) == 1.0 and hits_at_k([], [0.1, 0.2], 1) == 1.0
    g = fx.build_graph(fx.write_graph(str(tmp_path / "g")))
    torch.manual_seed(0)

    class Dot(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.u = torch.nn.Embedding(fx.N_USER, 8)
            self.i = torch.nn.Embedding(fx.N_ITEM, 8)

        def score(self, u, i):
            return (self.u(u) * self.i(i)).sum(-1)
    model = Dot()

    def train_ds():
        return gl.Dataset(g.E("buy").batch(16).shuffle(traverse=True).alias("pos").outV().alias("u").outNeg("buy").sample(4).by("random").alias("neg").values())

    def pos_ds():
        return gl.Dataset(g.E("buy").batch(32).alias("pos").values())

    def neg_ds():
        return gl.Dataset(g.V("user").batch(16).alias("u").outNeg("buy").sample(3).by("random").alias("neg").values())

    def step(m, b):
        e = b["pos"]
        u, i = e.tensor("src_ids"), e.tensor("dst_ids")
        neg = b["neg"].tensor("ids")
        pos_s = m.score(u, i)
        neg_s = m.score(u[:, None].expand_as(neg), neg)
        return F.softplus(-pos_s).mean() + F.softplus(neg_s).mean()

    def score(m, b):
        if "pos" in b:
            return m.score(b["pos"].tensor("src_ids"), b["pos"].tensor("dst_ids"))
        neg = b["neg"].tensor("ids")
        return m.score(b["u"].tensor("ids")[:, None].expand_as(neg), neg)
    tr = LinkDistTrainer(progress_steps=10000)
    before = tr.eval_hits(tr.eval(pos_ds(), model, score), tr.eval(neg_ds(), model, score), 10)["hits@10"]
    hist = tr.train_and_eval(train_ds(), model, step, pos_ds(), neg_ds(), score, learning_rate=5e-2, epochs=6, hit_K=10)
    assert len(hist) == 6 and hist[-1]["loss"] < hist[0]["loss"] and hist[-1]["hits@10"] > before + 0.15
    n = tr.predict(pos_ds(), model, lambda m, b: (b["pos"].tensor("src_ids"), b["pos"].tensor("dst_ids"),
                                                   m.score(b["pos"].tensor("src_ids"), b["pos"].tensor("dst_ids"))), str(tmp_path / "pred"))
    lines = open(str(tmp_path / "pred") + ".rank0").read().strip().split("\n")
    assert n == len(lines) - 1 == g.get_stats()["buy"][0] and lines[0].startswith("src_id:int64")


def test_nn_dataset_reference_methods(tmp_path):
    """nn.Dataset iteration / get_subgraphs(inducer) / get_subgraphs_v2(processor) and the TorchDataset compat surface of the
    reference's nn/pytorch Dataset (induce_func, as_dict, client_id, lazy_init)."""
    g = fx.build_graph(fx.write_graph(str(tmp_path)))
    q = g.V("item").batch(8).alias("s").outV("sim").sample(2).by("topk").alias("n").values()
    n_batches = sum(1 for _ in glnn.Dataset(q))
    assert n_batches == (fx.N_ITEM + 7) // 8
    first = next(glnn.Dataset(q).iterator)
    assert set(first) == {"s", "n"} and first["n"].floats.shape == (16, 4)

    class PairInducer(glnn.SubGraphInducer):
        def induce_func(self, values):
            src, nbr = values["s"], values["n"]
            pos = [(int(a), [int(x) for x in row]) for a, row in zip(src.ids.tolist(), nbr.ids.tolist())]
            return pos, None
    pos, neg = glnn.Dataset(q).get_subgraphs(PairInducer(use_neg=False))
    assert neg is None and len(pos) == 8 and all(len(r) == 2 for _, r in pos)

    class CountProcessor(glnn.SubGraphProcessor):
        def process_func(self, subgraph):
            return int(subgraph.num_nodes), tuple(subgraph.edge_index.shape)
    sq = g.SubGraph("item", "sim", batch_size=6).alias("sg").values()
    ds = glnn.Dataset(sq, batch_size=3)
    got = ds.get_subgraphs_v2(CountProcessor())
    assert len(got) == 3 and all(n == 6 and e[0] == 2 for n, e in got)
    total = 3
    with pytest.raises(gl.OutOfRangeError):
        while True:
            total += len(ds.get_subgraphs_v2(CountProcessor()))
    assert total == (fx.N_ITEM + 5) // 6
    # TorchDataset compat
    td = glnn.TorchDataset(q, induce_func=lambda d: [d["s"].ids.numel()])
    assert next(iter(td)) == [8] and not td.lazy_init()
    td.client_id = 3
    assert td.client_id == 3
    with pytest.raises(ValueError):
        td.client_id = "x"
    dd = next(iter(glnn.TorchDataset(q).as_dict()))
    assert isinstance(dd["s"], dict) and dd["s"]["ids"].shape == (8,) and dd["n"]["float_attrs"].shape == (16, 4)
    with pytest.raises(RuntimeError):
        glnn.TorchDataset(q, graph=gl.Graph())           # lazy client mode needs a launched server
    g.close()


def test_container_parity_methods():
    """BatchGraph.to_graphs, HeteroBatchGraph.from_graphs / transform / num_graphs / num_edges, TemporalGraph.hop_*, EgoLayer.append,
    SubGraph / HeteroSubGraph keys, GLError.message - method-level parity with the reference's containers."""
    ei = torch.cat([torch.tensor([[0, 1], [1, 2]]) + 3 * i for i in range(2)], 1)
    bg = glnn.BatchGraph(ei, glnn.Data(ids=torch.arange(6), floats=torch.arange(12.).reshape(6, 2)), graph_node_offsets=torch.tensor([0, 3, 6]))
    parts = bg.to_graphs()
    assert len(parts) == 2 and parts[1][0].tolist() == [[0, 1], [1, 2]] and parts[1][1].ids.tolist() == [3, 4, 5]
    assert bg.transform().to_graphs()[0][1].shape == (3, 2)
    hs = []
    for i in range(3):
        nodes = {"u": glnn.Data(ids=torch.arange(2) + 10 * i, floats=torch.ones(2, 3) * i), "v": glnn.Data(ids=torch.arange(4) + 100 * i, floats=torch.ones(4, 5))}
        hs.append(glnn.HeteroSubGraph({("u", "r", "v"): torch.tensor([[0, 3], [1, 0]])}, nodes))
    assert set(hs[0].keys) >= {"edge_index_dict", "nodes_dict"}
    hb = glnn.HeteroBatchGraph.from_graphs(hs)
    assert hb.num_graphs == 3 and hb.num_edges(("u", "r", "v")) == 6 and hb.num_nodes("v") == 12 and hb.node_types == ["u", "v"]
    # rows index the tail type (v: 4 per graph), cols the head type (u: 2 per graph)
    assert hb.edge_index_dict[("u", "r", "v")].tolist() == [[0, 3, 4, 7, 8, 11], [1, 0, 3, 2, 5, 4]]
    tr = hb.transform({"u": lambda d: d.floats * 2})
    assert tr.nodes_dict["u"].shape == (6, 3) and float(tr.nodes_dict["u"][4, 0]) == 4.0 and tr.nodes_dict["v"].shape == (12, 5)
    tg = glnn.TemporalGraph(glnn.Data(ids=torch.arange(2)), torch.tensor([5, 6]), [glnn.Data(ids=torch.arange(4))], [torch.tensor([1, 2, 3, 4])],
                            [glnn.Data(ids=torch.arange(4))], [2])
    assert tg.hop_node(0).ids.numel() == 4 and tg.hop_t(0).tolist() == [1, 2, 3, 4] and tg.hop_edge(0).ids.numel() == 4
    layer = glnn.EgoLayer([glnn.EgoSAGEConv(4, 8)])
    layer.append(glnn.EgoSAGEConv(4, 8))
    assert len(layer.convs) == 2
    err = gl.NotFoundError("no such node")
    assert err.message == "no such node" and isinstance(err, gl.BaseError)
