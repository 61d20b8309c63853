"""Batch normalisation of the hidden layers of the fused GraphSAGE trainers (EgoGraphSAGE(batch_norm=True)): the
normalised, dropped-out H and the running statistics against torch's BatchNorm1d called once per hop tensor; every
gradient against autograd; training parity with the autograd model; inference with the running statistics;
checkpoints; launch counts and the rejected configurations.

Collected after the other GPU tests on purpose: late in a long session torch.profiler was seen to drop the first kernel
of a profiled step, and the exact launch counts of the earlier files must not depend on this file's session time."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests.test_sage_agg_gpu import _csr_agg, _engine_routes, _ref, first_max_oracle  # noqa: F401  (fixture)
from tests.test_sage_dropout_gpu import _host_keep

pytestmark = pytest.mark.gpu

AGGS = ["mean", "sum", "max", "gcn"]


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


def _graph(rt, n, deg, feat, n_cls, seed, offset=0.0, noise=1.0):
    """labelled graph whose edges stay inside a class; features = offset + class centre * 0.5 + noise"""
    from graphlearn_b200.store.shards import CsrShard, IdMap, NodeTable
    dev = rt.device
    g = torch.Generator(device=dev).manual_seed(seed)
    labels = torch.randint(0, n_cls, (n,), device=dev, generator=g)
    x = torch.randn(n_cls, feat, device=dev, generator=g)[labels] * 0.5 + torch.randn(n, feat, device=dev, generator=g) * noise
    order = torch.argsort(labels)
    counts = torch.bincount(labels, minlength=n_cls)
    start = torch.cumsum(counts, 0) - counts
    src = torch.arange(n, device=dev).repeat_interleave(deg)
    c = labels[src]
    dst = order[start[c] + (torch.rand(src.numel(), device=dev, generator=g) * counts[c]).long().clamp(max=n - 1)]
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=dev), dense=True))
    nodes.set_float(x + offset, torch.float32)
    nodes.set_labels(labels)
    return nodes, CsrShard.from_coo(rt, "e", "n", "n", src, dst, n)


@pytest.fixture(scope="module")
def graph(rt):
    return _graph(rt, 30000, 20, 100, 47, seed=7)


def _model(rt, L, agg, out, p=0.0, hidden=256, in_dim=100, seed=0, **kw):
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    torch.manual_seed(seed)
    return EgoGraphSAGE(in_dim, hidden, out, L, agg_type=agg, dropout=p, batch_norm=True, **kw).to(rt.device)


def _fix_hops(tr, hops):
    """train on `hops` only, and keep the gradients and the weights (no optimiser, no counters)"""
    tr.sample = lambda s: hops
    tr.opt.advance = lambda *a, **k: None
    tr._skip_opt = True


def _keep(tr, l, p):
    seed, ctr = (int(x) for x in tr.drop_state.cpu())
    ly = tr.layers[l - 1]
    return _host_keep(seed, ctr, l, ly.rows, ly.conv.out_dim, p).to(ly.H.device)


def _oracle(model, tr, hops, fan, p, x=None):
    """EgoGNN with batch norm in torch (training mode: each hop tensor normalised with its own statistics, the running
    buffers updated once per hop tensor), each hidden hop tensor times the engine's dropout mask / (1 - p); layer 1
    reads the node table, or the dense rows `x` of every hop"""
    L = model.num_layers
    keeps = [_keep(tr, l, p) if p > 0 else None for l in range(1, L)]

    def hidden(l, z, i):
        h = torch.relu(model.norms[l](z))
        if p > 0:
            ly = tr.layers[l]
            h = h * keeps[l][ly.offs[i]:ly.offs[i + 1]].to(h.dtype) / (1 - p)
        return h.to(torch.bfloat16)

    def conv(l, a, b, i):
        if l == L - 1:
            return model.convs[l](a, b, fan[i])
        return hidden(l, model.convs[l](a, b, fan[i]), i)

    if x is None:
        h = [model.convs[0].forward_store(tr.nodes, hops[i], hops[i + 1], fan[i]) for i in range(L)]
        h = [hidden(0, z, i) for i, z in enumerate(h)] if L > 1 else h
    else:
        h = [conv(0, x[i], x[i + 1], i) for i in range(L)]
    for l in range(1, L):
        h = [conv(l, h[i], h[i + 1], i) for i in range(L - l)]
    return h[0].float()


def _sup_step(rt, nodes, csr, m, fan, B, seed=0, **kw):
    from graphlearn_b200.engine import FastSageTrainer
    tr = FastSageTrainer(rt, nodes, csr, m, fan, B, use_cuda_graph=False, **kw)
    seeds = torch.randint(0, nodes.n_local, (B,), device=rt.device, generator=torch.Generator(device=rt.device).manual_seed(seed))
    tr.seeds.copy_(seeds)
    hops = tr.sample(seeds)
    _fix_hops(tr, hops)
    return tr, hops


# ------------------------------------------------------------------------------------------------ 1. forward
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("L,fan,B", [(2, [25, 10], 512), (3, [5, 4, 3], 128)])
def test_bn_forward_matches_batchnorm1d(rt, graph, p, L, fan, B):
    """H of every BN layer = relu(BatchNorm1d(Z_s)) per segment on the engine's own Z, zero wherever the host Philox
    drops; the running buffers equal those of a BatchNorm1d called once per hop tensor in hop order"""
    nodes, csr = graph
    m = _model(rt, L, "mean", 47, p)
    norms0 = copy.deepcopy(m.norms)
    tr, hops = _sup_step(rt, nodes, csr, m, fan, B)
    if L == 3:
        assert tr.layers[1].ns > 1                     # the second layer's weight is N-split
    tr._step_body()
    torch.cuda.synchronize()
    for l, ly in enumerate(tr.layers[:-1], 1):
        ref = norms0[l - 1]
        keep = _keep(tr, l, p) if p > 0 else None
        for i in range(ly.nseg):
            rows = slice(ly.offs[i], ly.offs[i + 1])
            want = torch.relu(ref(ly.bn.Z[rows]))
            if p > 0:
                want = want * keep[rows] / (1 - p)
                assert bool((ly.H[rows][~keep[rows]] == 0).all()), (l, i)
            got = ly.H[rows].float()
            err = (got - want).abs().max()
            assert err <= 1e-2 * max(1.0, float(want.abs().max())), (l, i, float(err))
        bn = ly.bn.norm
        assert int(bn.num_batches_tracked) == int(ref.num_batches_tracked) == ly.nseg
        torch.testing.assert_close(bn.running_mean, ref.running_mean, rtol=1e-4, atol=1e-5)
        torch.testing.assert_close(bn.running_var, ref.running_var, rtol=1e-4, atol=1e-5)


def test_bn_variance_with_large_common_offset(rt):
    """features with |mean| >> std: the per-segment rstd of the engine equals the fp64 variance of its Z"""
    nodes, csr = _graph(rt, 20000, 20, 100, 8, seed=3, offset=1000.0, noise=8.0)
    m = _model(rt, 2, "mean", 8)
    tr, hops = _sup_step(rt, nodes, csr, m, [25, 10], 512)
    tr._step_body()
    torch.cuda.synchronize()
    ly = tr.layers[0]
    ratio = []
    for i in range(ly.nseg):
        z = ly.bn.Z[ly.offs[i]:ly.offs[i + 1]].double()
        var = z.var(0, unbiased=False)
        ratio.append(float((z.mean(0).abs() / var.sqrt()).median()))
        torch.testing.assert_close(ly.bn.mean[i].double(), z.mean(0), rtol=1e-6, atol=1e-4)
        torch.testing.assert_close(ly.bn.rstd[i].double(), 1 / (var + ly.bn.norm.eps).sqrt(), rtol=2e-4, atol=0)
    assert min(ratio) > 20, ratio


# ------------------------------------------------------------------------------------------------ 2. gradients
def _check_grads(m_fast, m_ref, max_tol, conv_tol=0.05, bn_tol=0.1):
    """Every conv parameter's gradient within `conv_tol` of the oracle's in norm, every BN parameter's within `bn_tol`, and the
    largest difference of any gradient entry within `max_tol` of the largest oracle entry.  d beta and d gamma are
    column sums over all rows of a layer whose terms largely cancel, so the bf16 rounding of dA and dY (in the engine)
    and of the activations (in both) weighs more in them: up to 6.4 % in norm for the first layer of the 3-layer
    models, against at most 5 % for the convs' weights."""
    errs = []
    for (name, a), b in zip(m_fast.named_parameters(), m_ref.parameters()):
        err = float((a.grad - b.grad).norm() / (b.grad.norm() + 1e-12))
        assert err < (bn_tol if name.startswith("norms.") else conv_tol), (name, err)
    g_fast = torch.cat([q.grad.reshape(-1) for q in m_fast.parameters()])
    g_ref = torch.cat([q.grad.reshape(-1) for q in m_ref.parameters()])
    rel = (g_fast - g_ref).abs().max() / (g_ref.abs().max() + 1e-8)
    assert rel < max_tol, float(rel)


def _grads_vs_autograd(rt, first_max_oracle, tr, m2, hops, fan, p, loss_fn, max_tol, x=None, conv_tol=0.05):  # noqa: F811
    tr._step_body()
    torch.cuda.synchronize()
    loss_fast = float(tr.loss)
    ly = tr.layers[0]
    if ly.argmax is not None:                          # layer 1 reads the learned table: route through its choices too
        first_max_oracle[id(m2.convs[0])] = [ly.argmax[ly.offs[i]:ly.offs[i + 1], :m2.convs[0].in_nbr].long()
                                             for i in range(ly.nseg)]
    _engine_routes(first_max_oracle, tr, m2)
    loss = loss_fn(_oracle(m2, tr, hops, fan, p, x))
    loss.backward()
    loss = float(loss.detach())
    assert abs(loss_fast - loss) < 2e-2 * max(1.0, abs(loss)), (loss_fast, loss)
    _check_grads(tr.model, m2, max_tol, conv_tol)
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("p", [0.0, 0.5])
@pytest.mark.parametrize("L,fan,B", [(2, [25, 10], 512), (3, [5, 4, 3], 128)])
def test_bn_gradients_match_autograd(rt, graph, first_max_oracle, agg, p, L, fan, B):  # noqa: F811
    nodes, csr = graph
    m1 = _model(rt, L, agg, 47, p)
    m2 = copy.deepcopy(m1)
    tr, hops = _sup_step(rt, nodes, csr, m1, fan, B)
    labels = nodes.labels.local[hops[0]]
    _grads_vs_autograd(rt, first_max_oracle, tr, m2, hops, fan, p, lambda o: F.cross_entropy(o, labels), 0.1)


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("kind", ["sigmoid", "softmax"])
@pytest.mark.parametrize("L,fan,p", [(2, [10, 5], 0.0), (3, [5, 4, 3], 0.5)])
def test_link_bn_gradients_match_autograd(rt, graph, first_max_oracle, agg, kind, L, fan, p):  # noqa: F811
    """the link trainer normalises each hop tensor over all R = B (2 + neg) roots' rows"""
    from graphlearn_b200.engine import FastLinkSageTrainer
    from tests.test_link_engine_gpu import _ref_loss
    nodes, csr = graph
    m1 = _model(rt, L, agg, 64, p)
    m2 = copy.deepcopy(m1)
    B, n, T = 128, 5, (0.5 if kind == "softmax" else 1.0)
    tr = FastLinkSageTrainer(rt, nodes, csr, m1, fan, B, n, loss=kind, temperature=T, use_cuda_graph=False)
    tr.seeds[:2 * B] = torch.randint(0, nodes.n_local, (2 * B,), device=rt.device)
    tr._draw_roots(tr.seeds)
    hops = tr.sample(tr.seeds)
    _fix_hops(tr, hops)
    tr._draw_roots = lambda r: None
    # (3 layers with dropout and BN: the single entries of the link model's gradients were seen to differ by up to 0.143
    # of the largest one, and W_1's gradient by 5.05 % in norm, against 0.1 / 0.12 and 5 % in the BN-free dropout tests)
    _grads_vs_autograd(rt, first_max_oracle, tr, m2, hops, fan, p, lambda o: _ref_loss(o, B, n, kind, T), 0.16,
                       conv_tol=0.06)


@pytest.mark.parametrize("agg", ["mean", "max"])
def test_bn_gradients_with_learned_input_embedding(rt, first_max_oracle, agg):  # noqa: F811
    """BN on layer 1 next to a learned input table: dZ_1 comes from the BN backward, and the table's gradient (dE)
    matches autograd"""
    from graphlearn_b200.engine import FastSageTrainer
    from tests.test_sage_embed_gpu import _featureless_graph, _gather
    nodes, csr = _featureless_graph(rt, 20000, 20, 8, seed=11)
    d, B, fan = 64, 256, [10, 5]
    m1 = _model(rt, 2, agg, 8, hidden=128, in_dim=d)
    m2 = copy.deepcopy(m1)
    tr = FastSageTrainer(rt, nodes, csr, m1, fan, B, learn_input_embedding=True, use_cuda_graph=False)
    seeds = torch.randint(0, nodes.n_local, (B,), device=rt.device)
    tr.seeds.copy_(seeds)
    hops = tr.sample(seeds)
    _fix_hops(tr, hops)
    with torch.no_grad():                              # the weights as the engine's bf16 images round them
        for c in m2.convs:
            c.weight_p.copy_(c.weight_p.bfloat16().float())
    E = tr.emb.table.local[:, :d].float().clone().requires_grad_(True)
    labels = nodes.labels.local[seeds]
    _grads_vs_autograd(rt, first_max_oracle, tr, m2, hops, fan, 0.0, lambda o: F.cross_entropy(o, labels), 0.1,
                       x=[_gather(E, h) for h in hops])
    g_ref = E.grad
    g = tr.emb.grad[:, :d]
    assert float((g - g_ref).norm() / g_ref.norm()) < 0.05
    assert float((g - g_ref).abs().max() / g_ref.abs().max()) < 0.1


# ------------------------------------------------------------------------------------------------- 3. training
def test_bn_training_tracks_autograd(rt, graph):
    """20 captured steps on the engine against the autograd EgoGraphSAGE(batch_norm=True) + Adam on the same batches:
    the losses, the parameters and the running statistics track"""
    nodes, csr = graph
    B, fan, steps, lr = 512, [25, 10], 20, 3e-3
    m1 = _model(rt, 2, "mean", 47)
    m2 = copy.deepcopy(m1)
    from graphlearn_b200.engine import FastSageTrainer
    tr = FastSageTrainer(rt, nodes, csr, m1, fan, B, lr=lr)
    sd = tr.state_dict()
    tr.capture()
    tr.load_state_dict(sd)                             # undo the warm-up steps (parameters and running statistics)
    g = torch.Generator(device=rt.device).manual_seed(1)
    batches, losses = [], []
    for t in range(steps):
        tr.step_device(torch.randint(0, nodes.n_local, (B,), device=rt.device, generator=g))
        torch.cuda.synchronize()
        batches.append([h.clone() for h in tr._hops[t & 1]])
        losses.append(float(tr.loss_out))
    opt = torch.optim.Adam(m2.parameters(), lr=lr)
    ref = []
    for hops in batches:
        opt.zero_grad()
        loss = F.cross_entropy(m2.forward_store(nodes, hops, fan), nodes.labels.local[hops[0]])
        loss.backward()
        opt.step()
        ref.append(float(loss))
    for a, b in zip(losses, ref):
        assert abs(a - b) < 0.03 * abs(b), (losses, ref)
    p1 = torch.cat([q.detach().reshape(-1) for q in m1.parameters()])
    p2 = torch.cat([q.detach().reshape(-1) for q in m2.parameters()])
    assert float((p1 - p2).norm() / p2.norm()) < 0.02
    for a, b in zip(m1.norms, m2.norms):
        assert int(a.num_batches_tracked) == int(b.num_batches_tracked) == 2 * steps
        assert float((a.running_mean - b.running_mean).norm() / b.running_mean.norm()) < 0.02
        assert float((a.running_var - b.running_var).norm() / b.running_var.norm()) < 0.02


@pytest.mark.parametrize("agg", AGGS)
def test_bn_training_learns_3layer(rt, agg):
    from graphlearn_b200.engine import FastSageTrainer
    from tests.test_sage_agg_gpu import _homophilous_graph
    nodes, csr = _homophilous_graph(rt, 20000, 20, 64, 8, seed=9)
    tr = FastSageTrainer(rt, nodes, csr, _model(rt, 3, agg, 8, hidden=128, in_dim=64), [5, 4, 3], 256, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    tr.capture()
    losses = []
    for _ in range(80):
        loss = tr.step(torch.randint(0, 20000, (256,)))
        torch.cuda.synchronize()
        losses.append(float(loss))
    assert all(x == x for x in losses)
    assert sum(losses[-5:]) / 5 < 0.6 * losses[0], (losses[0], losses[-5:])


# ------------------------------------------------------------------------------------------------ 4. inference
def _eval_oracle(tr):
    """fp32 eval-mode full-neighbourhood forward in torch (BN with the running statistics), bf16 hidden rounding"""
    from graphlearn_b200.ops import sage as S
    nodes, csr = tr.nodes, tr.csr
    h = nodes.feats.local[:, :nodes.float_dim].float()
    ar = torch.arange(h.size(0), device=h.device)
    for l, c in enumerate(tr.convs):
        last = l == len(tr.convs) - 1
        w = S.logical_weight(c.weight_p.detach(), c.in_self, c.in_nbr, c.agg_type)
        y = _ref(h, _csr_agg(h, csr.indptr.local, csr.indices.local, ar, c.agg_type), w,
                 None if c.bias is None else c.bias.detach(), False, c.agg_type)
        if not last:
            n = tr.model.norms[l]
            y = torch.relu(F.batch_norm(y, n.running_mean, n.running_var, n.weight, n.bias, False, 0.0, n.eps))
        h = y if last else y.bfloat16().float()
    return h


def _state(tr):
    return [t.clone() for n in tr.model.norms for t in (n.running_mean, n.running_var, n.num_batches_tracked)] + \
        [ly.img.clone() for ly in tr.layers] + [tr.flat_p.clone()]


@pytest.mark.parametrize("agg", ["mean", "max"])
@pytest.mark.parametrize("L,fan", [(2, [25, 10]), (3, [5, 4, 3])])
def test_bn_inference_uses_running_statistics(rt, graph, agg, L, fan):
    from graphlearn_b200.engine import FastSageTrainer
    nodes, csr = graph
    tr = FastSageTrainer(rt, nodes, csr, _model(rt, L, agg, 47, 0.5, seed=1), fan, 256, use_cuda_graph=False)
    for _ in range(5):
        tr.step(torch.randint(0, nodes.n_local, (256,)))
    torch.cuda.synchronize()
    before = _state(tr)
    got = tr.infer_all()
    torch.cuda.synchronize()
    ref = _eval_oracle(tr)
    # (the engine rounds the folded weights gamma / sigma W to bf16, the oracle rounds W and scales in fp32: 2.6 % of
    # the largest logit was seen for the 2-layer mean model, against the 2 % the BN-free inference tests allow)
    err = (got - ref).abs().max()
    assert err <= 4e-2 * ref.abs().max(), (float(err), float(ref.abs().max()))
    assert torch.equal(got, tr.infer_all())
    vids = torch.arange(0, nodes.n_local, 7, device=rt.device)
    acc = tr.evaluate(vids)
    want = float((got[vids].argmax(1) == nodes.labels.local[vids]).float().mean())
    assert acc == want
    # predict: the eval-mode autograd path on sampled hops, BN with the running statistics
    seeds = torch.randint(0, nodes.n_local, (64,), device=rt.device)
    hops = tr.sample(seeds)
    tr.sample = lambda s: hops
    out = tr.predict(seeds)
    m = tr.model
    with torch.no_grad():
        h = [m.convs[0].forward_store(nodes, hops[i], hops[i + 1], fan[i]) for i in range(L)]
        for l in range(L):
            if l > 0:
                h = [m.convs[l](h[i], h[i + 1], fan[i]) for i in range(L - l)]
            if l < L - 1:
                n = m.norms[l]
                h = [torch.relu(F.batch_norm(z, n.running_mean, n.running_var, n.weight, n.bias, False, 0.0, n.eps))
                     .bfloat16() for z in h]
    torch.testing.assert_close(out, h[0].float(), rtol=1e-3, atol=1e-3)
    assert m.training
    after = _state(tr)
    assert all(torch.equal(a, b) for a, b in zip(before, after))


# ----------------------------------------------------------------------------------------------- 5. checkpoint
def test_bn_checkpoint_round_trip(rt, graph):
    """a fresh trainer (other init, other seed) that loads a state dict computes the original's next step bit for bit
    (every hidden Z and H, the running buffers); a state dict without the BN state raises"""
    from graphlearn_b200.engine import FastSageTrainer
    nodes, csr = graph
    tr = FastSageTrainer(rt, nodes, csr, _model(rt, 3, "mean", 47, 0.5), [5, 4, 3], 256, use_cuda_graph=False)
    for _ in range(3):
        tr.step(torch.randint(0, nodes.n_local, (256,)))
    torch.cuda.synchronize()
    sd = tr.state_dict()
    tr2 = FastSageTrainer(rt, nodes, csr, _model(rt, 3, "mean", 47, 0.5, seed=5), [5, 4, 3], 256, seed=3,
                          use_cuda_graph=False)
    tr2.load_state_dict(sd)
    tr.repack()
    hops = tr.sample(torch.randint(0, nodes.n_local, (256,), device=rt.device))
    for t in (tr, tr2):
        _fix_hops(t, hops)
        t._step_body()
    torch.cuda.synchronize()
    for a, b in zip(tr.layers[:-1], tr2.layers[:-1]):
        assert torch.equal(a.bn.Z, b.bn.Z) and torch.equal(a.H, b.H)
        for k in ("running_mean", "running_var", "num_batches_tracked"):
            assert torch.equal(getattr(a.bn.norm, k), getattr(b.bn.norm, k)), k
    assert torch.equal(tr.layers[-1].H, tr2.layers[-1].H)
    old = {k: v for k, v in sd.items() if k != "batch_norm"}
    with pytest.raises(ValueError):
        tr2.load_state_dict(old)


# ------------------------------------------------------------------------------------------ 6. launch count
def test_bn_step_launch_count(rt, graph):
    """one BN layer adds 5 launches of this repo's kernels (forward: statistics, apply; backward: dY, sums, apply) and
    no library kernel: 14 supervised and 17 link launches for the 2-layer model, against the 9 and 12 without BN that
    tests/test_link_engine_gpu.py counts.  The steps with and without BN are profiled side by side (see the module
    docstring)."""
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from tests.test_link_engine_gpu import _count_launches
    nodes, csr = graph
    B = 128
    e = (torch.randint(0, nodes.n_local, (B,)), torch.randint(0, nodes.n_local, (B,)))
    counts = {}
    for bn in (False, True):
        sup = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2, batch_norm=bn).to(rt.device), [25, 10], 256,
                              use_cuda_graph=False)
        sup._step_body()
        tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 64, 2, batch_norm=bn).to(rt.device), [25, 10],
                                 B, 5, use_cuda_graph=False)
        tr.step(*e)
        counts[bn] = (_count_launches(sup._step_body), _count_launches(lambda: tr.step(*e)))
    for (own0, lib0, _), (own, lib, names) in zip(counts[False], counts[True]):
        assert lib0 == 0 and lib == 0, (lib0, lib)
        assert own == own0 + 5, (own0, own, names)
        for k in ("glb::bn_colsum_kernel<false>", "glb::bn_colsum_kernel<true>", "glb::bn_apply_kernel",
                  "glb::bn_bwd_apply_kernel", "glb::sage_bwd_dz_kernel<false>"):
            assert names.get(k) == 1, (k, names)


# --------------------------------------------------------------------------------------------- 7. rejections
def test_bn_rejections(rt, graph):
    from graphlearn_b200.engine import FastSageTrainer
    nodes, csr = graph
    with pytest.raises(ValueError):
        FastSageTrainer(rt, nodes, csr, _model(rt, 2, "mean", 47), [25, 10], 1, use_cuda_graph=False)
    for mom in (0.0, 1.5, -0.1):
        with pytest.raises(ValueError):
            _model(rt, 2, "mean", 47, bn_momentum=mom)
