"""GSL query -> static plan -> captured graph / fused engine (gsl/compile.py, FastSageTrainer.from_query)."""
import copy
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _write_tsv(d, n, deg, dim, ncls, seed=0):
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, ncls, (n,), generator=g)
    centers = torch.randn(ncls, dim, generator=g)
    x = centers[labels] * 0.5 + torch.randn(n, dim, generator=g)
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "node.tsv"), "w") as f:
        f.write("id:int64\tlabel:int32\tfeature:string\n")
        for i in range(n):
            f.write("%d\t%d\t%s\n" % (i, int(labels[i]), ":".join("%.4f" % v for v in x[i].tolist())))
    dst = torch.randint(0, n, (n, deg), generator=g)
    with open(os.path.join(d, "edge.tsv"), "w") as f:
        f.write("src_id:int64\tdst_id:int64\n")
        for i in range(n):
            for j in dst[i].tolist():
                f.write("%d\t%d\n" % (i, j))
    return d


@pytest.fixture(scope="module")
def tsv_graph(tmp_path_factory):
    import graphlearn_b200 as gl
    assert torch.cuda.is_available()
    d = _write_tsv(str(tmp_path_factory.mktemp("gsl_engine")), 3000, 12, 100, 7)
    gl.set_feature_dtype("bf16")
    g = gl.Graph()
    g.node(os.path.join(d, "node.tsv"), "i", decoder=gl.Decoder(labeled=True, attr_types=["float"] * 100))
    g.edge(os.path.join(d, "edge.tsv"), ("i", "i", "e"), decoder=gl.Decoder())
    g.init()
    return g


def _query(g, B=256, fan=(10, 5), traverse=True):
    q = g.V("i").batch(B).shuffle(traverse=traverse).alias("src")
    for i, k in enumerate(fan):
        q = q.outV("e").sample(k).by("random").alias("h%d" % (i + 1))
    return q.values()


def test_compiled_dataset_epochs_and_membership(tsv_graph):
    import graphlearn_b200 as gl
    from graphlearn_b200.gsl.compile import compile_query
    g = tsv_graph
    q = _query(g)
    plan = compile_query(q)
    assert plan is not None and plan.fanouts == [10, 5] and plan.traverse == "shuffle" and plan.batch_size == 256
    ds = gl.Dataset(q, window=4)
    assert ds.compiled
    csr = g.store.edges["e"]
    ip, idx = csr.indptr.local.cpu(), csr.indices.local.cpu()
    adj = {r: set(idx[ip[r]:ip[r + 1]].tolist()) for r in range(3000)}
    for epoch in range(2):
        seen = []
        while True:
            try:
                v = ds.next()
            except gl.OutOfRangeError:
                break
            src, h1, h2 = (torch.as_tensor(v[a].ids) for a in ("src", "h1", "h2"))      # .ids: numpy, like the reference
            assert h1.shape == (src.numel(), 10) and h2.shape == (src.numel() * 10, 5)
            for i in range(0, src.numel(), 37):
                assert set(h1[i].tolist()) <= adj[int(src[i])]
            flat1 = h1.reshape(-1)
            for i in range(0, flat1.numel(), 211):
                assert set(h2[i].tolist()) <= adj[int(flat1[i])]
            seen.append(src)
        allv = torch.cat(seen)
        assert allv.numel() == 3000 and torch.equal(torch.sort(allv).values, torch.arange(3000))   # traversed exactly once
    assert ds.epoch == 2
    # lazily fetched attributes of a compiled batch go through the normal lookup path
    v = ds.next()
    assert v["src"].labels.shape == (256,) and v["h1"].float_attrs.shape == (256, 10, 100)


def test_from_query_matches_raw_trainer(tsv_graph):
    """TSV -> gl.Graph -> GSL -> compiled plan -> fused engine == FastSageTrainer on the raw shards."""
    import graphlearn_b200 as gl
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.gsl.iterators import SeedIterator
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    g = tsv_graph
    rt = g.runtime
    torch.manual_seed(0)
    m1 = EgoGraphSAGE(100, 256, 7, 2).to(rt.device)
    m2 = copy.deepcopy(m1)
    q = _query(g)
    tr1 = FastSageTrainer.from_query(g, q, m1, lr=5e-3, seed=11)
    tr2 = FastSageTrainer(rt, g.store.nodes["i"], g.store.edges["e"], m2, [10, 5], 256, lr=5e-3, seed=11)
    tr1.capture(); tr2.capture()
    it = SeedIterator(3000, 256, "shuffle", "cpu", seed=gl.config.get().seed + 17 * rt.rank, drop_last=True)
    vids = torch.arange(3000)
    l1, l2 = [], []
    steps = 0
    for epoch in range(2):
        while True:
            try:
                a = tr1.step_query()
            except gl.OutOfRangeError:
                break
            b = tr2.step(vids[it.next_index()].clone())
            torch.cuda.synchronize()
            l1.append(float(a)); l2.append(float(b))
            steps += 1
        try:
            it.next_index()
        except gl.OutOfRangeError:
            pass
    assert steps == 2 * (3000 // 256) and tr1.epoch == 2
    # same kernels, same seeds, same RNG stream: equal up to the summation order of the split-K red.global.add
    # (the first steps agree to ~1e-6; Adam amplifies the rounding noise over the following steps)
    assert torch.allclose(torch.tensor(l1[:6]), torch.tensor(l2[:6]), rtol=1e-4, atol=1e-5), (l1[:6], l2[:6])
    assert torch.allclose(torch.tensor(l1), torch.tensor(l2), rtol=5e-2, atol=5e-3), (l1[-4:], l2[-4:])
    assert l1[-1] < l1[1]        # (pipelined step(): entry 0 reports the priming batch) - it learns


def test_dgs_kernels_match_cpu_service():
    """csrc/dgs.cu (one launch per record batch / per query hop) vs the portable torch implementation."""
    import numpy as np
    from graphlearn_b200.dgs import DynamicGraphService, QueryPlan
    schema = {"vertices": {"u": {"count": 500, "feat_dim": 4}, "i": {"count": 800, "feat_dim": 4}},
              "edges": {"click": {"src": "u", "dst": "i"}, "sim": {"src": "i", "dst": "i"}}}
    plan = lambda: QueryPlan("u").out("click", 6).out("sim", 3)   # noqa: E731
    a, b = DynamicGraphService(schema, device="cuda"), DynamicGraphService(schema, device="cpu")
    a.install_query(1, plan()); b.install_query(1, plan())
    rs = np.random.RandomState(1)
    t = 0
    for it in range(5):
        for et, ns in (("click", 500), ("sim", 800)):
            n = 4000
            src = (rs.zipf(1.4, n) % ns).astype(np.int64)            # hot sources: many records per vertex per batch
            dst = rs.randint(0, 800, n).astype(np.int64)
            ts = np.arange(t, t + n); t += n
            upd = {"edges": {et: {"src": src, "dst": dst, "ts": ts, "weight": rs.rand(n).astype(np.float32)}}}
            a.apply_updates(upd); b.apply_updates(upd)
    feat = rs.rand(800, 4).astype(np.float32)
    for s in (a, b):
        s.apply_updates({"vertices": {"i": {"id": np.arange(800), "ts": np.zeros(800, dtype=np.int64), "feat": feat}}})
    q = list(range(0, 500, 3)) + [499, 700000, -5]
    ra, rb = a.run_query(1, q), b.run_query(1, q)
    for h in range(2):
        assert torch.equal(ra["hops"][h]["timestamps"].cpu(), rb["hops"][h]["timestamps"])
        assert torch.equal(ra["hops"][h]["ids"].cpu(), rb["hops"][h]["ids"])
        assert torch.allclose(ra["hops"][h]["weights"].cpu(), rb["hops"][h]["weights"])
    assert torch.equal(a.stores["click"].count.cpu(), b.stores["click"].count)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_knn_fused_kernel_flat_and_ivf(dtype):
    """csrc/knn.cu: wgmma score GEMM + fused running top-k + merge; recall@k = 1.0 vs an fp32 brute force."""
    import graphlearn_b200 as gl
    from graphlearn_b200.ops import knn
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.shards import IdMap, NodeTable
    rt = init()
    g = torch.Generator(device=rt.device).manual_seed(5)
    n, d, B, k = 70001, 100, 300, 10
    x = torch.randn(n, d, device=rt.device, generator=g)
    t = NodeTable(rt, "t", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    t.set_float(x, dtype)
    xs = t.feats.local[:, :d].float()
    q = torch.randn(B, d, device=rt.device, generator=g)
    for metric in (0, 1):
        ids, dist = knn.search(rt, t, q, k, metric)
        sc = q @ xs.t() if metric == 1 else -torch.cdist(q, xs) ** 2
        ref_s, ref_i = torch.topk(sc, k, dim=1)
        assert torch.equal(torch.sort(ids, 1).values, torch.sort(ref_i, 1).values), metric       # recall 1.0
        want = ref_s if metric == 1 else -ref_s
        assert torch.allclose(dist, want, rtol=1e-3, atol=1e-2)
    # IVF-flat: probing every list is exact, probing a quarter keeps most of the neighbours
    opt = gl.IndexOption(); opt.index_type = "ivfflat"; opt.nlist = 64; opt.nprobe = 64
    knn.build_index(t, opt)
    ids, _ = knn.search(rt, t, q, k, 0)
    ref_i = torch.topk(-torch.cdist(q, xs) ** 2, k, dim=1).indices
    assert torch.equal(torch.sort(ids, 1).values, torch.sort(ref_i, 1).values)
    opt.nprobe = 16
    knn.build_index(t, opt)
    ids, _ = knn.search(rt, t, q[:64], k, 0)
    hit = (ids[:, :, None] == ref_i[:64, None, :]).any(2).float().mean()
    assert hit > 0.5, float(hit)


def test_knn_flat_wide_queries_single_slab_buffer():
    """256-wide queries leave shared memory for one database slab only: the flat scan then loads and scores the slabs
    one after the other, with recall 1.0 vs an fp32 brute force like the double-buffered scan."""
    from graphlearn_b200.ops import knn
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.shards import IdMap, NodeTable
    rt = init()
    g = torch.Generator(device=rt.device).manual_seed(6)
    n, d, B, k = 20001, 256, 200, 10
    x = torch.randn(n, d, device=rt.device, generator=g)
    t = NodeTable(rt, "t", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    t.set_float(x, torch.bfloat16)
    xs = t.feats.local[:, :d].float()
    q = torch.randn(B, d, device=rt.device, generator=g)
    for metric in (0, 1):
        ids, _ = knn.search(rt, t, q, k, metric)
        sc = q @ xs.t() if metric == 1 else -torch.cdist(q, xs) ** 2
        ref_i = torch.topk(sc, k, dim=1).indices
        assert torch.equal(torch.sort(ids, 1).values, torch.sort(ref_i, 1).values), metric


@pytest.mark.parametrize("dtype,d,H,k", [(torch.bfloat16, 100, 4, 10), (torch.float32, 64, 2, 7), (torch.bfloat16, 256, 4, 25)])
def test_gat_fused_kernels(dtype, d, H, k):
    """csrc/gat.cu: gather + online-softmax attention aggregation (fwd) and its backward vs the torch oracle, both reading
    a feature store (layer 1) and dense activations (deeper layers); then the whole EgoGATConv vs the literal reference."""
    from graphlearn_b200.nn.conv import EgoGATConv
    from graphlearn_b200.ops import gat as GAT
    from graphlearn_b200.parallel.runtime import init
    from graphlearn_b200.store.shards import IdMap, NodeTable
    rt = init()
    g = torch.Generator(device=rt.device).manual_seed(3)
    n, M = 5000, 333
    t = NodeTable(rt, "t", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    t.set_float(torch.randn(n, d, device=rt.device, generator=g), dtype)
    feats = t.feats.local[:, :d].float()
    sv = torch.randint(0, n, (M,), device=rt.device, generator=g)
    nv = torch.randint(0, n, (M * k,), device=rt.device, generator=g)
    u_x = (torch.randn(H, d, device=rt.device, generator=g) * 0.2).requires_grad_()
    u_n = (torch.randn(H, d, device=rt.device, generator=g) * 0.2).requires_grad_()
    c = torch.randn(H, device=rt.device, generator=g).requires_grad_()
    # ---- store inputs
    a = GAT.gat_aggregate(u_x, u_n, c, k=k, self_table=t, self_vids=sv, nbr_table=t, nbr_vids=nv)
    go = torch.randn(a.shape, device=rt.device, generator=g)
    (a.float() * go).sum().backward()
    u2 = [p.detach().clone().requires_grad_() for p in (u_x, u_n, c)]
    ref = GAT.gat_aggregate_reference(u2[0], u2[1], u2[2], feats[sv], feats[nv], k)
    (ref * go.to(torch.bfloat16).float()).sum().backward()
    assert (a.float() - ref).abs().max() < 3e-2 * ref.abs().max()
    for p_, q_, name in zip((u_x, u_n, c), u2, "xnc"):
        rel = (p_.grad - q_.grad).abs().max() / (q_.grad.abs().max() + 1e-6)
        assert rel < 5e-2, (name, float(rel))
    # ---- dense inputs with input gradients
    xs = feats[sv].to(dtype).requires_grad_()
    xn = feats[nv].to(dtype).requires_grad_()
    for p_ in (u_x, u_n, c):
        p_.grad = None
    a = GAT.gat_aggregate(u_x, u_n, c, k=k, x_self=xs, x_nbr=xn)
    (a.float() * go).sum().backward()
    xs2, xn2 = xs.detach().float().requires_grad_(), xn.detach().float().requires_grad_()
    ref = GAT.gat_aggregate_reference(u_x.detach(), u_n.detach(), c.detach(), xs2, xn2, k)
    (ref * go.to(torch.bfloat16).float()).sum().backward()
    for p_, q_, name in ((xs, xs2, "xs"), (xn, xn2, "xn")):
        rel = (p_.grad.float() - q_.grad).abs().max() / (q_.grad.abs().max() + 1e-6)
        assert rel < 5e-2, (name, float(rel))
    # ---- the layer: fused path == literal reference layer
    conv = EgoGATConv(d, 64, num_head=H, use_bias=True).to(rt.device).eval()
    y = conv.forward_store(t, sv, nv, k)
    y_ref = conv.forward_reference(feats[sv], feats[nv], k)
    assert (y - y_ref).abs().max() < 3e-2 * max(1.0, float(y_ref.abs().max()))


def test_graphed_train_step_matches_eager():
    """engine/graphed.py: forward + loss + backward + Adam captured once; replays train exactly like the eager step."""
    from graphlearn_b200.engine.graphed import GraphedTrainStep
    from graphlearn_b200.parallel.runtime import init
    rt = init()
    from graphlearn_b200.nn.conv import EgoGATConv
    from graphlearn_b200.store.shards import IdMap, NodeTable
    n, d, k = 3000, 32, 6
    g = torch.Generator(device=rt.device).manual_seed(0)
    tab = NodeTable(rt, "t", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    tab.set_float(torch.randn(n, d, device=rt.device, generator=g), torch.bfloat16)
    target = torch.randn(n, 16, device=rt.device, generator=g)

    def make():
        torch.manual_seed(1)
        conv = EgoGATConv(d, 16, num_head=2).to(rt.device)
        opt = torch.optim.Adam(conv.parameters(), lr=1e-2, capturable=True)

        def loss_fn(v):
            out = conv.forward_store(tab, v["s"], v["n"], k)
            return ((out.float() - target[v["s"]]) ** 2).mean()
        return conv, opt, loss_fn

    batches = [{"s": torch.randint(0, n, (256,), device=rt.device, generator=g),
                "n": torch.randint(0, n, (256 * k,), device=rt.device, generator=g)} for _ in range(8)]
    conv_e, opt_e, loss_e = make()
    eager = []
    for b in batches[:1] * 3 + batches:             # the graphed step warms up 3x on its example batch
        opt_e.zero_grad(set_to_none=True)
        l = loss_e(b); l.backward(); opt_e.step()
        eager.append(float(l))
    conv_g, opt_g, loss_g = make()
    step = GraphedTrainStep(loss_g, opt_g, batches[0], warmup=3)
    got = [float(step(b)) for b in batches]
    assert step.replays == 8 and step.eager_steps == 0
    assert torch.allclose(torch.tensor(got), torch.tensor(eager[3:]), rtol=2e-3, atol=1e-5), (got, eager[3:])
    short = {"s": batches[0]["s"][:100], "n": batches[0]["n"][:100 * k]}
    assert float(step(short)) > 0 and step.eager_steps == 1          # other shapes fall back to the eager step
