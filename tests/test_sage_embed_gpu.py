"""Fused GraphSAGE training on featureless nodes with a learned layer-1 input embedding (learn_input_embedding=True): the
scattered embedding gradient and the touched-row bitmap against autograd, the lazy Adam update against
torch.optim.SparseAdam, training parity with an autograd baseline, checkpoints, launch counts and rejected
configurations."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests.test_sage_agg_gpu import _csr_agg, _engine_routes, _ref, first_max_oracle  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

AGGS = ["mean", "sum", "max", "gcn"]


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


def _featureless_graph(rt, n, deg, n_cls, seed):
    """labelled graph without float attributes whose edges stay inside a class (the labels are its communities)"""
    from graphlearn_b200.store.shards import CsrShard, IdMap, NodeTable
    dev = rt.device
    g = torch.Generator(device=dev).manual_seed(seed)
    labels = torch.randint(0, n_cls, (n,), device=dev, generator=g)
    order = torch.argsort(labels)
    counts = torch.bincount(labels, minlength=n_cls)
    start = torch.cumsum(counts, 0) - counts
    src = torch.arange(n, device=dev).repeat_interleave(deg)
    c = labels[src]
    dst = order[start[c] + (torch.rand(src.numel(), device=dev, generator=g) * counts[c]).long().clamp(max=n - 1)]
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=dev), dense=True))
    nodes.set_labels(labels)
    assert nodes.float_dim == 0 and nodes.feat_desc is None
    return nodes, CsrShard.from_coo(rt, "e", "n", "n", src, dst, n)


@pytest.fixture(scope="module")
def graph(rt):
    return _featureless_graph(rt, 20000, 20, 8, seed=11)


def _model(rt, d, hidden, out, L, agg, seed=0):
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    torch.manual_seed(seed)
    return EgoGraphSAGE(d, hidden, out, L, agg_type=agg).to(rt.device)


def _sup(rt, graph, model, fan, B, **kw):
    from graphlearn_b200.engine import FastSageTrainer
    return FastSageTrainer(rt, *graph, model, fan, B, learn_input_embedding=True, **kw)


def _link(rt, graph, model, fan, B, neg, **kw):
    from graphlearn_b200.engine import FastLinkSageTrainer
    return FastLinkSageTrainer(rt, *graph, model, fan, B, neg, learn_input_embedding=True, **kw)


def _bitmap_rows(bits, n):
    w = bits.long() & 0xFFFFFFFF
    return ((w[:, None] >> torch.arange(32, device=bits.device)) & 1).flatten()[:n].bool()


def _gather(E, h):
    """rows of E for the ids h; ids outside the table read a zero row"""
    n = E.size(0)
    Ez = torch.cat([E, torch.zeros(1, E.size(1), device=E.device, dtype=E.dtype)])
    return Ez[torch.where((h >= 0) & (h < n), h, torch.full_like(h, n))]


# --------------------------------------------------------------------------- 1. gradient and bitmap vs autograd
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("L,fan", [(2, [10, 5]), (3, [5, 4, 3])])
@pytest.mark.parametrize("link", [False, True], ids=["supervised", "link"])
def test_embedding_gradient_matches_autograd(rt, graph, first_max_oracle, agg, L, fan, link):
    from tests.test_link_engine_gpu import _ref_loss
    nodes = graph[0]
    n, d = nodes.n_local, 64
    m1 = _model(rt, d, 128, 32 if link else 8, L, agg)
    m2 = copy.deepcopy(m1)
    if link:
        B, neg = 128, 5
        tr = _link(rt, graph, m1, fan, B, neg, use_cuda_graph=False)
        tr.seeds[:2 * B] = torch.randint(0, n, (2 * B,), device=rt.device)
        tr._draw_roots(tr.seeds)
        tr._draw_roots = lambda r: None
        hops = tr.sample(tr.seeds)
    else:
        B = 256
        tr = _sup(rt, graph, m1, fan, B, use_cuda_graph=False)
        seeds = torch.randint(0, n, (B,), device=rt.device)
        tr.seeds.copy_(seeds)
        hops = tr.sample(seeds)
    hops[-1][:40] = -1                                    # ids outside the table: zero rows, no gradient, no bit
    tr.sample = lambda s: hops
    tr.opt.advance = lambda *a, **k: None
    tr._skip_opt = True
    tr._step_body()
    torch.cuda.synchronize()
    e = tr.emb
    # oracle: the dense model over rows gathered from an fp32 copy of the table layer 1 read, with the weights rounded
    # as the engine's bf16 images round them (EgoSAGEConv's dense max path multiplies by the fp32 weights; the ReLU
    # masks that difference flips show in single entries of a row gradient that sums a few routed columns)
    with torch.no_grad():
        for c in m2.convs:
            c.weight_p.copy_(c.weight_p.bfloat16().float())
    E = e.table.local[:, :d].float().clone().requires_grad_(True)
    if agg == "max":                                  # route every layer through the engine's argmax choices
        ly = tr.layers[0]
        first_max_oracle[id(m2.convs[0])] = [ly.argmax[ly.offs[i]:ly.offs[i + 1], :d].long() for i in range(ly.nseg)]
        _engine_routes(first_max_oracle, tr, m2)
    out = m2([_gather(E, h) for h in hops], fan)
    if link:
        loss = _ref_loss(out, B, neg, "sigmoid", 1.0)
    else:
        loss = F.cross_entropy(out, nodes.labels.local[hops[0]])
    loss.backward()
    assert abs(float(tr.loss) - float(loss)) < 2e-2 * max(1.0, abs(float(loss))), (float(tr.loss), float(loss))
    g_ref, g = E.grad, e.grad[:, :d]
    norm_err = float((g - g_ref).norm() / g_ref.norm())
    max_err = float((g - g_ref).abs().max() / g_ref.abs().max())
    assert norm_err < 0.05, norm_err
    # (max hands a column's whole gradient to one child; the link loss sharpens it: see test_sage_agg_gpu)
    assert max_err < (0.08 if agg == "max" and link else 0.05), max_err
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]
    read = torch.zeros(n, dtype=torch.bool, device=rt.device)
    for h in hops:
        v = h[(h >= 0) & (h < n)]
        read[v] = True
    assert torch.equal(_bitmap_rows(e.bits, n), read)


# --------------------------------------------------------------------------- 2. lazy Adam vs SparseAdam
@pytest.mark.parametrize("agg", ["mean", "max"])
def test_lazy_adam_matches_sparse_adam(rt, graph, agg):
    nodes = graph[0]
    n, d = nodes.n_local, 64
    tr = _sup(rt, graph, _model(rt, d, 128, 8, 2, agg), [10, 5], 256, use_cuda_graph=False, embedding_lr=0.02)
    e, o = tr.emb, tr.opt
    ref = torch.nn.Embedding(n, e.master.size(1), sparse=True).to(rt.device)
    with torch.no_grad():
        ref.weight.copy_(e.master)
    sopt = torch.optim.SparseAdam([ref.weight], lr=e.lr, betas=o.betas, eps=o.eps)
    for step in range(3):
        tr._skip_opt = True
        tr.step(torch.randint(0, n, (256,)))               # advances the Adam step, keeps the gradient and the bitmap
        torch.cuda.synchronize()
        touched = _bitmap_rows(e.bits, n)
        rows = touched.nonzero().flatten()
        grad, before = e.grad.clone(), e.master.clone()
        assert int(touched.sum()) > 1000 and int(o.step_t) == step + 1
        assert bool((grad[~touched] == 0).all())
        tr.C.embed_lazy_adam(e.master, e.m, e.v, e.grad, e.table.local, e.bits, o.step_t, e.lr, o.betas[0], o.betas[1],
                             o.eps)
        tr.g_store.zero_()                                 # (the dense update was skipped)
        torch.cuda.synchronize()
        ref.weight.grad = torch.sparse_coo_tensor(rows[None], grad[rows], ref.weight.shape)
        sopt.step()
        torch.testing.assert_close(e.master[rows], ref.weight.detach()[rows], rtol=2e-6, atol=1e-7)
        assert torch.equal(e.master[~touched], before[~touched])
        assert torch.equal(e.table.local[:, :e.master.size(1)], e.master.to(torch.bfloat16))
        assert int(e.bits.abs().sum()) == 0 and int(e.grad.abs().sum()) == 0
    st = sopt.state[ref.weight]
    torch.testing.assert_close(e.m, st["exp_avg"].to_dense() if st["exp_avg"].is_sparse else st["exp_avg"],
                               rtol=2e-6, atol=1e-9)
    torch.testing.assert_close(e.v, st["exp_avg_sq"].to_dense() if st["exp_avg_sq"].is_sparse else st["exp_avg_sq"],
                               rtol=2e-6, atol=1e-12)


def test_initialisation_is_a_seeded_truncated_normal(rt, graph):
    d = 64
    a = _sup(rt, graph, _model(rt, d, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False, seed=4)
    b = _sup(rt, graph, _model(rt, d, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False, seed=4)
    c = _sup(rt, graph, _model(rt, d, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False, seed=5)
    E = a.input_embedding()
    assert E.shape == (graph[0].n_local, d) and E.dtype == torch.float32
    assert torch.equal(E, b.input_embedding()) and not torch.equal(E, c.input_embedding())
    s = d ** -0.5
    assert float(E.abs().max()) <= 2 * s
    # a normal truncated at +-2 sigma has std 0.880 sigma
    assert abs(float(E.std()) / s - 0.880) < 0.01, float(E.std()) / s
    assert torch.equal(a.emb.table.local[:, :d], E.to(torch.bfloat16))


# --------------------------------------------------------------------------- 3. training parity with autograd
def _snapshot_captured(tr, steps, roots_fn):
    """run `steps` captured device-only steps from the trainer's state at the call (capture's eager warm-up steps are
    undone); returns the hop lists each step trained on and the engine's losses"""
    sd = tr.state_dict()
    tr.capture()
    tr.load_state_dict(sd)
    hops, losses = [], []
    for t in range(steps):
        tr.step_device(*roots_fn(t))
        torch.cuda.synchronize()
        hops.append([h.clone() for h in tr._hops[t & 1]])
        losses.append(float(tr.loss_out))
    return hops, losses


def _baseline(rt, model, E0, lr, emb_lr, batches, loss_fn):
    """autograd: nn.Embedding(sparse=True) + SparseAdam for E, the dense model + Adam, on the engine's batches"""
    emb = torch.nn.Embedding(E0.size(0), E0.size(1), sparse=True).to(rt.device)
    with torch.no_grad():
        emb.weight.copy_(E0)
    o1 = torch.optim.SparseAdam([emb.weight], lr=emb_lr)
    o2 = torch.optim.Adam(model.parameters(), lr=lr)
    losses = []
    for hops in batches:
        o1.zero_grad(); o2.zero_grad()
        loss = loss_fn(model([emb(h) for h in hops], [len(h) // len(p) for p, h in zip(hops, hops[1:])]), hops)
        loss.backward()
        o1.step(); o2.step()
        losses.append(float(loss))
    return emb.weight.detach(), losses


def _full_forward(convs, E, csr):
    """layer-wise full-neighbourhood forward of the trained model over E (what infer_all computes)"""
    from graphlearn_b200.ops import sage as S
    h = E.float()
    ar = torch.arange(h.size(0), device=h.device)
    for l, c in enumerate(convs):
        last = l == len(convs) - 1
        w = S.logical_weight(c.weight_p.detach(), c.in_self, c.in_nbr, c.agg_type)
        y = _ref(h, _csr_agg(h, csr.indptr.local, csr.indices.local, ar, c.agg_type), w, c.bias.detach(), not last,
                 c.agg_type)
        h = y if last else y.bfloat16().float()
    return h


def test_supervised_training_matches_autograd_baseline(rt, graph):
    nodes, csr = graph
    n, d, B, steps = nodes.n_local, 64, 256, 150
    lr, emb_lr = 5e-3, 2e-2
    m1 = _model(rt, d, 128, 8, 2, "mean")
    m2 = copy.deepcopy(m1)
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(0))
    train, held = perm[:n * 4 // 5], perm[n * 4 // 5:].to(rt.device)
    g = torch.Generator().manual_seed(1)
    tr = _sup(rt, graph, m1, [10, 5], B, lr=lr, embedding_lr=emb_lr)
    E0 = tr.input_embedding().clone()
    batches, _ = _snapshot_captured(tr, steps, lambda t: (train[torch.randint(0, train.numel(), (B,), generator=g)]
                                                          .to(rt.device),))
    acc = tr.evaluate(held)
    labels = nodes.labels.local
    E, _ = _baseline(rt, m2, E0, lr, emb_lr, batches, lambda out, hops: F.cross_entropy(out, labels[hops[0]]))
    with torch.no_grad():
        acc_ref = float((_full_forward(m2.convs, E, csr)[held].argmax(1) == labels[held]).float().mean())
    assert acc > 0.5 and acc_ref > 0.5, (acc, acc_ref)          # 8 classes: chance is 0.125
    assert abs(acc - acc_ref) <= 0.03, (acc, acc_ref)


def test_link_training_matches_autograd_baseline(rt, graph):
    from tests.test_link_engine_gpu import _ref_loss
    nodes, csr = graph
    n, d, B, neg, steps = nodes.n_local, 64, 128, 5, 150
    lr, emb_lr = 5e-3, 2e-2
    m1 = _model(rt, d, 128, 32, 2, "mean")
    m2 = copy.deepcopy(m1)
    tr = _link(rt, graph, m1, [10, 5], B, neg, lr=lr, embedding_lr=emb_lr)
    E0 = tr.input_embedding().clone()
    g = torch.Generator().manual_seed(2)
    rows = torch.arange(n, device=rt.device).repeat_interleave(csr.indptr.local[1:] - csr.indptr.local[:-1])
    cols = csr.indices.local

    def edges(t):
        i = torch.randint(0, cols.numel(), (B,), generator=g).to(rt.device)
        return rows[i], cols[i]
    batches, losses = _snapshot_captured(tr, steps, edges)
    _, ref = _baseline(rt, m2, E0, lr, emb_lr, batches, lambda out, hops: _ref_loss(out, B, neg, "sigmoid", 1.0))
    first, last = sum(ref[:10]) / 10, sum(ref[-10:]) / 10
    got_first, got_last = sum(losses[:10]) / 10, sum(losses[-10:]) / 10
    assert last < 0.8 * first and got_last < 0.8 * got_first, (first, last, got_first, got_last)
    assert abs(got_last - last) <= 0.1 * last, (got_last, last)


def test_predict_reads_the_learned_table(rt):
    """with every neighbour drawn, the sampled predict / embed equal infer_all over the learned table"""
    from graphlearn_b200.store.shards import CsrShard, IdMap, NodeTable
    n, dev = 5000, rt.device
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=dev), dense=True))
    nodes.set_labels(torch.randint(0, 8, (n,), device=dev))
    src = torch.arange(n, device=dev).repeat_interleave(10)
    csr = CsrShard.from_coo(rt, "e", "n", "n", src, torch.randint(0, n, (src.numel(),), device=dev), n)
    vids = torch.arange(0, n, 3, device=dev)
    for link in (False, True):
        m = _model(rt, 64, 128, 32 if link else 8, 2, "mean")
        kw = dict(strategy="random_without_replacement", use_cuda_graph=False)
        tr = _link(rt, (nodes, csr), m, [10, 10], 128, 3, **kw) if link else _sup(rt, (nodes, csr), m, [10, 10], 128, **kw)
        sampled = (tr.embed(vids) if link else tr.predict(vids)).float()
        full = tr.infer_all()[vids]
        assert float((sampled - full).abs().max()) <= 3e-2 * float(sampled.abs().max())


# --------------------------------------------------------------------------- 4. checkpoints
def test_checkpoint_resumes_embedding_training(rt, graph):
    n = graph[0].n_local
    batches = [torch.randint(0, n, (256,), generator=torch.Generator().manual_seed(i)) for i in range(4)]
    a = _sup(rt, graph, _model(rt, 64, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    for b in batches[:3]:
        a.step(b)
    torch.cuda.synchronize()
    sd = a.state_dict()
    b_ = _sup(rt, graph, _model(rt, 64, 128, 8, 2, "mean", seed=3), [10, 5], 256, use_cuda_graph=False, seed=9)
    b_.load_state_dict(sd)
    assert torch.equal(b_.emb.table.local, a.emb.table.local)
    for t in (a, b_):
        t.step(batches[3])
    torch.cuda.synchronize()
    for x, y in ((a.emb.master, b_.emb.master), (a.emb.m, b_.emb.m), (a.emb.v, b_.emb.v), (a.flat_p, b_.flat_p)):
        torch.testing.assert_close(x, y)
    with pytest.raises(ValueError):
        b_.load_state_dict({k: v for k, v in sd.items() if k != "input_embedding"})


# --------------------------------------------------------------------------- 5. launches and errors
def test_embedding_step_launch_count(rt, graph):
    """12 (supervised) / 15 (link) launches of this repository's kernels, no library kernel"""
    from tests.test_link_engine_gpu import _count_launches
    n = graph[0].n_local
    sup = _sup(rt, graph, _model(rt, 64, 128, 8, 2, "mean"), [15, 10], 256, use_cuda_graph=False)
    sup.seeds.copy_(torch.randint(0, n, (256,), device=rt.device))
    sup._step_body()
    s_own, s_lib, s_names = _count_launches(sup._step_body)
    B = 128
    tr = _link(rt, graph, _model(rt, 64, 128, 32, 2, "mean"), [15, 10], B, 5, use_cuda_graph=False)
    e = (torch.randint(0, n, (B,)), torch.randint(0, n, (B,)))
    tr.step(*e)
    own, lib, names = _count_launches(lambda: tr.step(*e))
    assert s_lib == 0 and lib == 0, (s_lib, lib)
    assert s_own == 12, s_names
    assert own == 15, names
    for nm in (s_names, names):
        assert nm.get("glb::embed_grad_scatter_kernel") == 1 and nm.get("glb::embed_lazy_adam_kernel") == 1, nm


def test_rejected_configurations(rt, graph):
    from graphlearn_b200.nn.conv import EgoSAGEConv
    from graphlearn_b200.store.synthetic import make_sharded_graph
    feat = make_sharded_graph(rt, 5000, 50000, 64, 8, seed=1)
    with pytest.raises(ValueError, match="float attributes"):
        _sup(rt, feat, _model(rt, 64, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    m = _model(rt, 64, 128, 8, 2, "mean")
    m.convs[0] = EgoSAGEConv((64, 32), 128, "mean").to(rt.device)
    with pytest.raises(ValueError, match="input widths"):
        _sup(rt, graph, m, [10, 5], 256, use_cuda_graph=False)
    with pytest.raises(ValueError, match="fused layer"):            # 64-wide bf16 rows: fan-outs up to 15
        _sup(rt, graph, _model(rt, 64, 128, 8, 2, "mean"), [20, 5], 256, use_cuda_graph=False)
