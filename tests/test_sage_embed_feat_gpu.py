"""Fused GraphSAGE training on node features concatenated with a learned per-node embedding (learn_input_embedding=True
on a node table with float attributes): layer 1 reads [E || x].  The scattered gradient of E and the gradient of W_1
against autograd, the combined bf16 image, dA_1 over E's column blocks only (sage_bwd_da with block ranges), the lazy
Adam update, training parity with an autograd baseline, inference, checkpoints, launch counts and rejected
configurations."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests.test_sage_agg_gpu import _engine_routes, _ref, first_max_oracle  # noqa: F401  (fixture)
from tests.test_sage_embed_gpu import _bitmap_rows, _featureless_graph, _gather, _model, _snapshot_captured

pytestmark = pytest.mark.gpu

AGGS = ["mean", "sum", "max", "gcn"]
D = 64                                              # width of E in every test


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


def _feat_graph(rt, f, dtype=torch.bfloat16, n=20000, seed=11):
    """the class-community graph of test_sage_embed_gpu with f float attributes: class centre * 0.5 + noise"""
    nodes, csr = _featureless_graph(rt, n, 20, 8, seed=seed)
    g = torch.Generator(device=rt.device).manual_seed(seed + 1)
    centers = torch.randn(8, f, device=rt.device, generator=g)
    x = centers[nodes.labels.local] * 0.5 + torch.randn(n, f, device=rt.device, generator=g)
    nodes.set_float(x, dtype)
    return nodes, csr


@pytest.fixture(scope="module")
def graphs(rt):
    cache = {}

    def get(f=100, dtype=torch.bfloat16):
        if (f, dtype) not in cache:
            cache[(f, dtype)] = _feat_graph(rt, f, dtype)
        return cache[(f, dtype)]
    return get


def _x(nodes):
    """the node table's attributes as layer 1 reads them: fp32 values of the bf16 rounding"""
    from graphlearn_b200.ops.gather import gather_rows
    return gather_rows(nodes.rt, nodes.feats, nodes.feat_desc, nodes.idmap.local_vids(), nodes.float_dim).bfloat16()


def _sup(rt, graph, model, fan, B, **kw):
    from graphlearn_b200.engine import FastSageTrainer
    return FastSageTrainer(rt, *graph, model, fan, B, learn_input_embedding=True, **kw)


def _link(rt, graph, model, fan, B, neg, **kw):
    from graphlearn_b200.engine import FastLinkSageTrainer
    return FastLinkSageTrainer(rt, *graph, model, fan, B, neg, learn_input_embedding=True, **kw)


@pytest.fixture
def bf16_a_tile(monkeypatch):
    """``sage_layer``'s fp32 reference path with the [self || aggregate] tile rounded to bf16 as the engine's A tile is
    (straight-through gradient).  A 164-wide layer 1 has K = 512, whose fused autograd op does not fit in shared memory
    next to 128 outputs, so the dense oracle's mean / sum layer 1 takes that path; unrounded, the ReLU masks its output
    flips against the engine's show in single entries of the gradient of E."""
    from graphlearn_b200.ops import sage as S

    def reference(weight, bias, xs, xn, k, mode="mean", relu=False):
        xn3 = xn.view(xs.size(0), k, -1).float()
        xs = xs.float()
        if mode == "gcn":
            a = (xs + xn3.sum(1)) / (k + 1)
        else:
            a = torch.cat([xs, xn3.mean(1) if mode == "mean" else xn3.sum(1)], 1)
        a = a + (a.bfloat16().float() - a).detach()
        y = F.linear(a, weight.float(), None if bias is None else bias.float())
        return F.relu(y) if relu else y
    monkeypatch.setattr(S, "sage_layer_reference", reference)


def _mean_forward(convs, x, csr):
    """layer-wise full-neighbourhood forward of a mean-aggregation model over the input rows x (what infer_all
    computes): A = [h || mean of the CSR row], rounded to bf16, bf16 weights, hidden layers ReLU -> bf16"""
    from graphlearn_b200.ops import sage as S
    indptr, indices = csr.indptr.local, csr.indices.local
    n = indptr.numel() - 1
    deg = indptr[1:] - indptr[:-1]
    row = torch.repeat_interleave(torch.arange(n, device=x.device), deg)
    h = x.float()
    for l, c in enumerate(convs):
        last = l == len(convs) - 1
        agg = torch.zeros(n, h.size(1), dtype=torch.float64, device=x.device).index_add_(0, row, h.double()[indices])
        agg = (agg / deg.clamp(min=1).double()[:, None]).float()
        w = S.logical_weight(c.weight_p.detach(), c.in_self, c.in_nbr, c.agg_type)
        y = _ref(h[:n], agg, w, c.bias.detach(), not last, "mean")
        h = y if last else y.bfloat16().float()
    return h


def _close(g, g_ref, max_tol):
    norm_err = float((g - g_ref).norm() / g_ref.norm())
    max_err = float((g - g_ref).abs().max() / g_ref.abs().max())
    assert norm_err < 0.05, norm_err
    assert max_err < max_tol, max_err


# --------------------------------------------------------------------------- 1. gradients of E and W_1 vs autograd
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("L,fan", [(2, [10, 5]), (3, [5, 4, 3])])
@pytest.mark.parametrize("link", [False, True], ids=["supervised", "link"])
def test_gradients_match_autograd(rt, graphs, first_max_oracle, bf16_a_tile, agg, L, fan, link):
    from tests.test_link_engine_gpu import _ref_loss
    graph = graphs()
    nodes = graph[0]
    n, f = nodes.n_local, nodes.float_dim
    m1 = _model(rt, D + f, 128, 32 if link else 8, L, agg)
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
    assert (e.d, e.f) == (D, f)
    # oracle: the dense model over rows [E_fp32 || bf16(x)] with the engine's bf16 weight rounding
    with torch.no_grad():
        for c in m2.convs:
            c.weight_p.copy_(c.weight_p.bfloat16().float())
    E = e.master[:, :D].bfloat16().float().clone().requires_grad_(True)
    X = _x(nodes).float()
    if agg == "max":                                  # route every layer through the engine's argmax choices
        ly = tr.layers[0]
        first_max_oracle[id(m2.convs[0])] = [ly.argmax[ly.offs[i]:ly.offs[i + 1], :D + f].long() for i in range(ly.nseg)]
        _engine_routes(first_max_oracle, tr, m2)
    out = m2([_gather(torch.cat([E, X], 1), h) for h in hops], fan)
    if link:
        loss = _ref_loss(out, B, neg, "sigmoid", 1.0)
    else:
        loss = F.cross_entropy(out, nodes.labels.local[hops[0]])
    loss.backward()
    assert abs(float(tr.loss) - float(loss)) < 2e-2 * max(1.0, abs(float(loss))), (float(tr.loss), float(loss))
    tol = 0.08 if agg == "max" and link else 0.05
    _close(e.grad[:, :D], E.grad, tol)
    # W_1 with its attribute columns (the dW kernel reads them from the saved A tile, not from dA_1)
    _close(m1.convs[0].weight_p.grad, m2.convs[0].weight_p.grad, tol)
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]
    read = torch.zeros(n, dtype=torch.bool, device=rt.device)
    for h in hops:
        read[h[(h >= 0) & (h < n)]] = True
    assert torch.equal(_bitmap_rows(e.bits, n), read)


# --------------------------------------------------------------------------- 2. the combined image
@pytest.mark.parametrize("f", [50, 100])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_image_holds_embedding_then_attributes(rt, graphs, f, dtype):
    graph = graphs(f, dtype)
    nodes = graph[0]
    n = nodes.n_local
    tr = _sup(rt, graph, _model(rt, D + f, 128, 8, 2, "mean"), [10, 5], 256)
    e = tr.emb
    img = e.table.local
    x = _x(nodes)
    assert e.view.float_dim == D + f and int(e.desc[1]) == D + f
    assert torch.equal(img[:, D:D + f], x)
    assert torch.equal(img[:, :D], e.master[:, :D].bfloat16())
    assert int(img[:, D + f:].float().abs().sum()) == 0            # row padding
    E0 = tr.input_embedding().clone()
    g = torch.Generator().manual_seed(3)
    _snapshot_captured(tr, 50, lambda t: (torch.randint(0, n, (256,), generator=g).to(rt.device),))
    assert not torch.equal(tr.input_embedding(), E0)
    assert torch.equal(img[:, D:D + f].view(torch.int16), x.view(torch.int16))
    assert torch.equal(img[:, :D], e.master[:, :D].bfloat16())
    assert int(img[:, D + f:].float().abs().sum()) == 0


# --------------------------------------------------------------------------- 3. dA over a window of column blocks
@pytest.mark.parametrize("rows,n_out,kt,n_imgs,N,ranges", [
    (3000, 128, 512, 1, 128, [(0, 1)]),                 # one range
    (3000, 128, 512, 1, 128, [(0, 1), (4, 5)]),         # E's blocks of the self and the neighbour half
    (1000, 47, 256, 1, 64, [(3, 4), (0, 2)]),           # two ranges, the second one first
    (16384, 256, 512, 4, 64, [(1, 3), (5, 6)]),         # N-split layer: 4 images, many row blocks per CTA
])
def test_windowed_da_matches_full_launch(rt, rows, n_out, kt, n_imgs, N, ranges):
    from graphlearn_b200.parallel.runtime import native
    C = native()
    g = torch.Generator(device=rt.device).manual_seed(rows + n_out)
    R = n_imgs * N
    wpad = torch.zeros(R, kt, device=rt.device)
    wpad[:n_out] = torch.randn(n_out, kt, device=rt.device, generator=g) / kt ** 0.5
    img = torch.cat([C.pack_weight_f32(wpad[i * N:(i + 1) * N].contiguous(), N, False)[0] for i in range(n_imgs)])
    dzp = torch.zeros(rows, R, dtype=torch.bfloat16, device=rt.device)
    dzp[:, :n_out] = torch.randn(rows, n_out, device=rt.device, generator=g).to(torch.bfloat16)
    full = torch.full((rows, kt), float("nan"), dtype=torch.bfloat16, device=rt.device)
    C.sage_bwd_da(dzp, img, N, n_imgs, full, 1.5)
    sentinel = torch.tensor(-1234.0, dtype=torch.bfloat16)
    win = torch.full((rows, kt), float(sentinel), dtype=torch.bfloat16, device=rt.device)
    C.sage_bwd_da(dzp, img, N, n_imgs, win, 1.5, ranges)
    torch.cuda.synchronize()
    inside = torch.zeros(kt, dtype=torch.bool, device=rt.device)
    for lo, hi in ranges:
        inside[lo * 64:hi * 64] = True
    assert torch.isfinite(full.float()).all()
    assert torch.equal(win[:, inside].view(torch.int16), full[:, inside].view(torch.int16))
    assert bool((win[:, ~inside] == sentinel.to(rt.device)).all())


def test_layer1_da_covers_only_embedding_blocks(rt, graphs):
    """layer 1 passes E's blocks of each half (gcn: its one half); the other layers, and f = 0, pass none"""
    graph = graphs()
    f = graph[0].float_dim                                          # 164 columns: each half pads to 256 = 4 blocks
    for agg, want in (("mean", ((0, 1), (4, 5))), ("gcn", ((0, 1),))):
        tr = _sup(rt, graph, _model(rt, D + f, 128, 8, 2, agg), [10, 5], 256, use_cuda_graph=False)
        assert tr.layers[0].da_blocks == want and tr.layers[1].da_blocks == ()
    bare = _featureless_graph(rt, 2000, 10, 8, seed=1)
    tr = _sup(rt, bare, _model(rt, D, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    assert tr.layers[0].da_blocks == ()


# --------------------------------------------------------------------------- 4. lazy Adam vs SparseAdam
def test_lazy_adam_matches_sparse_adam(rt, graphs):
    graph = graphs()
    nodes = graph[0]
    n, f = nodes.n_local, nodes.float_dim
    tr = _sup(rt, graph, _model(rt, D + f, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False, embedding_lr=0.02)
    e, o = tr.emb, tr.opt
    x = e.table.local[:, D:D + f].clone()
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
        tr.C.embed_lazy_adam(e.master, e.m, e.v, e.grad, e.table.local, e.bits, o.step_t, e.lr, o.betas[0], o.betas[1],
                             o.eps)
        tr.g_store.zero_()                                 # (the dense update was skipped)
        torch.cuda.synchronize()
        ref.weight.grad = torch.sparse_coo_tensor(rows[None], grad[rows], ref.weight.shape)
        sopt.step()
        torch.testing.assert_close(e.master[rows], ref.weight.detach()[rows], rtol=2e-6, atol=1e-7)
        assert torch.equal(e.master[~touched], before[~touched])
        assert torch.equal(e.table.local[:, :D], e.master.to(torch.bfloat16))
        assert torch.equal(e.table.local[:, D:D + f], x)
        assert int(e.bits.abs().sum()) == 0 and int(e.grad.abs().sum()) == 0


# --------------------------------------------------------------------------- 5. training parity with autograd
def _baseline(rt, model, E0, X, lr, emb_lr, batches, loss_fn):
    """autograd: nn.Embedding(sparse=True) + SparseAdam for E, rows [E || x], the dense model + Adam, on the engine's
    batches"""
    emb = torch.nn.Embedding(E0.size(0), E0.size(1), sparse=True).to(rt.device)
    with torch.no_grad():
        emb.weight.copy_(E0)
    o1 = torch.optim.SparseAdam([emb.weight], lr=emb_lr)
    o2 = torch.optim.Adam(model.parameters(), lr=lr)
    losses = []
    for hops in batches:
        o1.zero_grad(); o2.zero_grad()
        rows = [torch.cat([emb(h), X[h]], 1) for h in hops]
        loss = loss_fn(model(rows, [len(h) // len(p) for p, h in zip(hops, hops[1:])]), hops)
        loss.backward()
        o1.step(); o2.step()
        losses.append(float(loss))
    return emb.weight.detach(), losses


def test_supervised_training_matches_autograd_baseline(rt):
    # weak attributes (centre * 0.1): the learned embedding has to carry part of the signal
    nodes, csr = _featureless_graph(rt, 20000, 20, 8, seed=11)
    f = 48
    g0 = torch.Generator(device=rt.device).manual_seed(5)
    nodes.set_float(torch.randn(8, f, device=rt.device, generator=g0)[nodes.labels.local] * 0.1
                    + torch.randn(nodes.n_local, f, device=rt.device, generator=g0), torch.bfloat16)
    graph = (nodes, csr)
    n, B, steps = nodes.n_local, 256, 150
    lr, emb_lr = 5e-3, 2e-2
    m1 = _model(rt, D + f, 128, 8, 2, "mean")
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
    X = _x(nodes).float()
    E, _ = _baseline(rt, m2, E0, X, lr, emb_lr, batches, lambda out, hops: F.cross_entropy(out, labels[hops[0]]))
    with torch.no_grad():
        acc_ref = float((_mean_forward(m2.convs, torch.cat([E, X], 1), csr)[held].argmax(1) == labels[held])
                        .float().mean())
    assert acc > 0.5 and acc_ref > 0.5, (acc, acc_ref)          # 8 classes: chance is 0.125
    assert abs(acc - acc_ref) <= 0.03, (acc, acc_ref)


def test_link_training_matches_autograd_baseline(rt, graphs):
    from tests.test_link_engine_gpu import _ref_loss
    graph = graphs()
    nodes, csr = graph
    n, f, B, neg, steps = nodes.n_local, nodes.float_dim, 128, 5, 150
    lr, emb_lr = 5e-3, 2e-2
    m1 = _model(rt, D + f, 128, 32, 2, "mean")
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
    _, ref = _baseline(rt, m2, E0, _x(nodes).float(), lr, emb_lr, batches,
                       lambda out, hops: _ref_loss(out, B, neg, "sigmoid", 1.0))
    first, last = sum(ref[:10]) / 10, sum(ref[-10:]) / 10
    got_first, got_last = sum(losses[:10]) / 10, sum(losses[-10:]) / 10
    assert last < 0.9 * first and got_last < 0.9 * got_first, (first, last, got_first, got_last)
    assert abs(got_last - last) <= 0.1 * last, (got_last, last)


# --------------------------------------------------------------------------- 6. inference
def test_predict_and_embed_read_the_combined_image(rt):
    """with every neighbour drawn, the sampled predict / embed equal infer_all over [E || x]"""
    from graphlearn_b200.store.shards import CsrShard, IdMap, NodeTable
    n, f, dev = 5000, 100, rt.device
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=dev), dense=True))
    nodes.set_labels(torch.randint(0, 8, (n,), device=dev))
    nodes.set_float(torch.randn(n, f, device=dev), torch.bfloat16)
    src = torch.arange(n, device=dev).repeat_interleave(10)
    csr = CsrShard.from_coo(rt, "e", "n", "n", src, torch.randint(0, n, (src.numel(),), device=dev), n)
    vids = torch.arange(0, n, 3, device=dev)
    for link in (False, True):
        m = _model(rt, D + f, 128, 32 if link else 8, 2, "mean")
        kw = dict(strategy="random_without_replacement", use_cuda_graph=False)
        tr = _link(rt, (nodes, csr), m, [10, 10], 128, 3, **kw) if link else _sup(rt, (nodes, csr), m, [10, 10], 128, **kw)
        sampled = (tr.embed(vids) if link else tr.predict(vids)).float()
        full = tr.infer_all()[vids]
        assert float((sampled - full).abs().max()) <= 3e-2 * float(sampled.abs().max())
        with torch.no_grad():                           # and infer_all is the layer-wise forward over [E || bf16(x)]
            ref = _mean_forward(m.convs, torch.cat([tr.input_embedding().bfloat16().float(), _x(nodes).float()], 1),
                                csr)
        assert float((full - ref[vids]).abs().max()) <= 3e-2 * float(ref.abs().max())


# --------------------------------------------------------------------------- 7. checkpoints
def test_checkpoint_resumes_training(rt, graphs):
    graph = graphs()
    n, f = graph[0].n_local, graph[0].float_dim
    batches = [torch.randint(0, n, (256,), generator=torch.Generator().manual_seed(i)) for i in range(4)]
    a = _sup(rt, graph, _model(rt, D + f, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    for b in batches[:3]:
        a.step(b)
    torch.cuda.synchronize()
    sd = a.state_dict()
    assert sd["input_embedding"]["master"].shape == (n, D)
    b_ = _sup(rt, graph, _model(rt, D + f, 128, 8, 2, "mean", seed=3), [10, 5], 256, use_cuda_graph=False, seed=9)
    b_.load_state_dict(sd)
    assert torch.equal(b_.emb.table.local, a.emb.table.local)
    for t in (a, b_):
        t.step(batches[3])
    torch.cuda.synchronize()
    for x, y in ((a.emb.master, b_.emb.master), (a.emb.m, b_.emb.m), (a.emb.v, b_.emb.v), (a.flat_p, b_.flat_p)):
        torch.testing.assert_close(x, y)
    # the whole image: the attribute columns and the padding bit for bit; E's columns are the bf16 rounding of masters
    # that agree up to the order of the gradient scatter's fp32 reductions, so a rounding boundary may fall between them
    ia, ib = a.emb.table.local, b_.emb.table.local
    assert torch.equal(ib[:, D:], ia[:, D:])
    assert torch.equal(ib[:, :D], b_.emb.master[:, :D].bfloat16())
    torch.testing.assert_close(ib[:, :D].float(), ia[:, :D].float(), rtol=2 ** -7, atol=1e-6)


# --------------------------------------------------------------------------- 8. launches
def _kernels(names):
    """kernel name -> launches, template arguments dropped (layer 1's persistent-kernel instantiation follows its width)"""
    out = {}
    for k, v in names.items():
        out[k.split("<")[0]] = out.get(k.split("<")[0], 0) + v
    return out


def test_step_launch_count(rt, graphs):
    """12 (supervised) / 15 (link) launches of this repository's kernels, the featureless embedding step's kernels, no
    library kernel"""
    from tests.test_link_engine_gpu import _count_launches
    feat = graphs()
    bare = _featureless_graph(rt, 20000, 20, 8, seed=11)
    n, f = feat[0].n_local, feat[0].float_dim
    got = {}
    for key, graph, width in (("feat", feat, D + f), ("bare", bare, D)):
        sup = _sup(rt, graph, _model(rt, width, 128, 8, 2, "mean"), [15, 10], 256, use_cuda_graph=False)
        sup.seeds.copy_(torch.randint(0, n, (256,), device=rt.device))
        sup._step_body()
        s_own, s_lib, s_names = _count_launches(sup._step_body)
        B = 128
        tr = _link(rt, graph, _model(rt, width, 128, 32, 2, "mean"), [15, 10], B, 5, use_cuda_graph=False)
        e = (torch.randint(0, n, (B,)), torch.randint(0, n, (B,)))
        tr.step(*e)
        own, lib, names = _count_launches(lambda: tr.step(*e))
        assert s_lib == 0 and lib == 0, (s_lib, lib)
        assert s_own == 12, s_names
        assert own == 15, names
        got[key] = (_kernels(s_names), _kernels(names))
    assert got["feat"] == got["bare"], got


# --------------------------------------------------------------------------- 9. rejected configurations
def test_rejected_configurations(rt, graphs):
    from graphlearn_b200.nn.conv import EgoSAGEConv
    graph = graphs()
    f = graph[0].float_dim
    with pytest.raises(ValueError, match="float attributes"):          # no columns left for E
        _sup(rt, graph, _model(rt, f, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    with pytest.raises(ValueError, match="multiple of 8"):             # d = 60: the fp32 tables' padding would overwrite x
        _sup(rt, graph, _model(rt, f + 60, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    fp8 = _feat_graph(rt, 100, torch.float8_e4m3fn, n=2000)
    with pytest.raises(ValueError, match="fp8"):
        _sup(rt, fp8, _model(rt, D + 100, 128, 8, 2, "mean"), [10, 5], 256, use_cuda_graph=False)
    m = _model(rt, D + f, 128, 8, 2, "mean")
    m.convs[0] = EgoSAGEConv((D + f, D + f - 8), 128, "mean").to(rt.device)
    with pytest.raises(ValueError, match="input widths"):
        _sup(rt, graph, m, [10, 5], 256, use_cuda_graph=False)
    with pytest.raises(ValueError, match="fused layer"):                # 164-wide bf16 rows: fan-outs up to 63
        _sup(rt, graph, _model(rt, D + f, 128, 8, 2, "mean"), [64, 5], 256, use_cuda_graph=False)
