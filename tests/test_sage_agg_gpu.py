"""GraphSAGE with max and gcn aggregation on the fused CUDA engine: the sampled and CSR modes of the persistent kernel
(with the argmax bytes of max) against a torch oracle, bit-exact on integer data, the fused trainers' gradients against
autograd, captured training, layer-wise inference and launch counts."""
import copy

import pytest
import torch
import torch.nn.functional as F

from tests.test_sage_inference_gpu import DTYPES, SPECIAL_DEGREES, _csr, _degrees, _table

pytestmark = pytest.mark.gpu

AGGS = ["max", "gcn"]


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


@pytest.fixture
def first_max_oracle(monkeypatch):
    """EgoSAGEConv's dense max path with explicit gradient routing: each column's gradient goes to ONE neighbour, the
    first maximal one (torch.argmax; torch's max(dim) backward may pick any maximal index on CUDA), or, where the test
    registers them in the returned dict (id(conv) -> index tensors per call), the neighbours the engine's forward picked.
    Hidden activations of the engine and of the oracle differ in the last bf16 bit, which may flip the max of two
    nearly equal neighbours; routing through the engine's choice compares the backward alone (the choice itself is
    checked bit-exact against torch.argmax by test_max_exact_on_integers_and_argmax).  The dict's "agree" list collects
    the share of columns where the engine's choice is the oracle's own argmax."""
    from graphlearn_b200.nn import conv as conv_mod
    orig = conv_mod.EgoSAGEConv.forward
    routes = {"agree": []}

    def forward(self, x, neighbor, expand, relu=False, out_bf16=False):
        if self.agg_type != "max":
            return orig(self, x, neighbor, expand, relu, out_bf16)
        xn3 = neighbor.view(-1, expand, neighbor.size(-1)).float()
        idx = xn3.argmax(1, keepdim=True)
        q = routes.get(id(self))
        if q:
            eng = q.pop(0)[:, None, :]
            routes["agree"].append(float((eng == idx).float().mean()))
            idx = eng
        agg = xn3.gather(1, idx).squeeze(1)
        y = F.linear(torch.cat([x.float(), agg], 1), self.weight, self.bias)
        y = F.relu(y) if relu else y
        return y.to(torch.bfloat16) if out_bf16 else y
    monkeypatch.setattr(conv_mod.EgoSAGEConv, "forward", forward)
    return routes


def _engine_routes(routes, tr, model):
    """register the engine's argmax choices of layers >= 2 for the oracle copy `model` (same hop-pair call order)"""
    for ly, c in zip(tr.layers[1:], model.convs[1:]):
        if ly.argmax is not None:
            routes[id(c)] = [ly.argmax[ly.offs[i]:ly.offs[i + 1], :c.in_nbr].long() for i in range(ly.nseg)]


def _images(w, d, mode, N):
    from graphlearn_b200.ops import sage as S
    return S.pack_images(S.pad_weight(w, d, d, mode), N, 1)


def _ref(xs, agg, w, b, relu, mode):
    """the A tile rounded to bf16, bf16 weights, fp32 GEMM; gcn: A = the mean over {x} U nbrs only"""
    a = agg if mode == "gcn" else torch.cat([xs, agg], 1)
    y = F.linear(a.bfloat16().float(), w.bfloat16().float(), b)
    return F.relu(y) if relu else y


# ------------------------------------------------------------------------------------------- 1. sampled mode
def _sampled_layer(rt, nodes, self_vids, nbr_vids, k, w, b, mode, relu, out_bf16, amax=None):
    from graphlearn_b200.ops import sage as S
    from graphlearn_b200.parallel.runtime import native
    M, n_out, d = self_vids.numel(), w.size(0), nodes.float_dim
    N = S.pad_n(n_out)
    out = torch.full((M, n_out), 7.0, device=rt.device, dtype=torch.bfloat16 if out_bf16 else torch.float32)
    native().sage_fused_multi(nodes.feat_desc, nodes.feat_desc, [self_vids], [nbr_vids], [0], [0], [M], [k], [out], [None],
                              S.MODE[mode], _images(w, d, mode, N), b, N, n_out, relu, out_bf16, [], 1, 1,
                              [] if amax is None else [amax])
    torch.cuda.synchronize()
    return out.float()


def _sampled_agg(x, self_vids, nbr_vids, k, mode):
    """(x_self, aggregate, [M, k, d] neighbour rows); a -1 id reads a zero row"""
    xz = torch.cat([x, torch.zeros(1, x.size(1), device=x.device)])
    xn3 = xz[nbr_vids.view(-1, k)]
    xs = x[self_vids]
    agg = xn3.max(1).values if mode == "max" else (xs + xn3.sum(1)) / (k + 1)
    return xs, agg, xn3


@pytest.mark.parametrize("mode", AGGS)
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("d", [16, 100, 128, 256])
@pytest.mark.parametrize("k", [1, 4, 10, 25])
def test_sampled_layer_matches_oracle(rt, mode, dt, d, k):
    from graphlearn_b200.ops import sage as S
    n, M, n_out = 3000, 700, 47
    if not S.fused_supported(d, d, n_out, mode, k, torch.uint8 if dt == "fp8" else DTYPES[dt]):
        pytest.skip("k + 1 row pointers per row exceed the gather warp's scratch at this width")
    relu, out_bf16 = [(False, False), (True, True), (True, False), (False, True)][[16, 100, 128, 256].index(d)]
    g = torch.Generator(device=rt.device).manual_seed(d * 13 + k + len(mode))
    nodes, x = _table(rt, torch.randn(n, d, device=rt.device, generator=g), DTYPES[dt])
    self_vids = torch.randint(0, n, (M,), device=rt.device, generator=g)
    nbr_vids = torch.randint(0, n, (M * k,), device=rt.device, generator=g)
    nbr_vids[torch.rand(M * k, device=rt.device, generator=g) < 0.1] = -1
    w = torch.randn(n_out, d if mode == "gcn" else 2 * d, device=rt.device, generator=g) / (2 * d) ** 0.5
    b = torch.randn(n_out, device=rt.device, generator=g) * 0.1
    got = _sampled_layer(rt, nodes, self_vids, nbr_vids, k, w, b, mode, relu, out_bf16)
    xs, agg, _ = _sampled_agg(x, self_vids, nbr_vids, k, mode)
    ref = _ref(xs, agg, w, b, relu, mode)
    if out_bf16:
        ref = ref.bfloat16().float()
    err = (got - ref).abs().max()
    assert err <= 2e-2 * ref.abs().max() + 1e-3, (float(err), float(ref.abs().max()))


# ---------------------------------------------------------------------------------- 2. max, bit-exact + argmax
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("d", [16, 100, 256])
@pytest.mark.parametrize("k", [1, 4, 7, 13, 25])
def test_max_exact_on_integers_and_argmax(rt, dt, d, k):
    """Features and weights in {-1, 0, 1}: the max is exact, the A tile holds it exactly and the GEMM is exact in fp32,
    so the output equals the oracle bit for bit.  Three values over k rows tie all the time: the argmax bytes must be
    torch.argmax's first maximal index (k = 7 and 13 also end in a partial batch of row loads)."""
    from graphlearn_b200.ops import sage as S
    n, M, n_out = 2000, 600, 40
    if not S.fused_supported(d, d, n_out, "max", k, DTYPES[dt]):
        pytest.skip("k + 1 row pointers per row exceed the gather warp's scratch at this width")
    g = torch.Generator(device=rt.device).manual_seed(d + 100 * k)
    nodes, x = _table(rt, torch.randint(-1, 2, (n, d), device=rt.device, generator=g).float(), DTYPES[dt])
    self_vids = torch.randint(0, n, (M,), device=rt.device, generator=g)
    nbr_vids = torch.randint(0, n, (M * k,), device=rt.device, generator=g)
    nbr_vids[torch.rand(M * k, device=rt.device, generator=g) < 0.1] = -1
    w = torch.randint(-1, 2, (n_out, 2 * d), device=rt.device, generator=g).float()
    b = torch.randint(-3, 4, (n_out,), device=rt.device, generator=g).float()
    ld = (d + 15) // 16 * 16
    amax_rows = torch.full((M, ld + 16), 255, dtype=torch.uint8, device=rt.device)
    amax = amax_rows[:, :ld]
    got = _sampled_layer(rt, nodes, self_vids, nbr_vids, k, w, b, "max", False, False, amax=amax)
    xs, agg, xn3 = _sampled_agg(x, self_vids, nbr_vids, k, "max")
    ref = _ref(xs, agg, w, b, False, "max")
    assert torch.equal(got, ref), float((got - ref).abs().max())
    assert torch.equal(amax[:, :d].long(), xn3.argmax(1))
    assert bool((amax_rows[:, ld:] == 255).all())                     # nothing beyond the row is written


# ------------------------------------------------------------------------------------------------ 3. CSR mode
def _csr_agg(x, indptr, indices, self_vids, mode):
    n = indptr.numel() - 1
    deg = indptr[1:] - indptr[:-1]
    row = torch.repeat_interleave(torch.arange(n, device=x.device), deg)
    xv = x.double()[indices]
    if mode == "max":
        agg = torch.zeros(n, x.size(1), dtype=torch.float64, device=x.device)
        agg = agg.index_reduce_(0, row, xv, "amax", include_self=False)
    else:
        agg = torch.zeros(n, x.size(1), dtype=torch.float64, device=x.device).index_add_(0, row, xv)
        agg = (agg + x.double()[self_vids]) / (deg + 1).double()[:, None]
    return agg.float()


def _csr_layer(rt, nodes, indptr, indices, w, b, mode, relu, out_bf16, hub_degree=None):
    from graphlearn_b200.ops import sage as S
    n, d, n_out = nodes.n_local, nodes.float_dim, w.size(0)
    N = S.pad_n(n_out)
    plan = S.CsrPlan(indptr, indices, n, **({} if hub_degree is None else {"hub_degree": hub_degree}))
    out = torch.full((n, n_out), 7.0, device=rt.device, dtype=torch.bfloat16 if out_bf16 else torch.float32)
    plan.layer(nodes.feat_desc, nodes.feat_desc, torch.arange(n, device=rt.device), out, mode, _images(w, d, mode, N), b,
               N, n_out, relu, out_bf16)
    torch.cuda.synchronize()
    return out.float(), plan


@pytest.mark.parametrize("mode", AGGS)
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("d", [16, 100, 128, 256])
def test_csr_layer_max_gcn_matches_oracle(rt, mode, dt, d):
    n, n_out = 2000, 47
    relu, out_bf16 = [(False, False), (True, True), (True, False), (False, True)][[16, 100, 128, 256].index(d)]
    g = torch.Generator(device=rt.device).manual_seed(d * 5 + len(mode))
    nodes, x = _table(rt, torch.randn(n, d, device=rt.device, generator=g), DTYPES[dt])
    indptr, indices = _csr(rt, _degrees(n, d), n, d)
    w = torch.randn(n_out, d if mode == "gcn" else 2 * d, device=rt.device, generator=g) / (2 * d) ** 0.5
    b = torch.randn(n_out, device=rt.device, generator=g) * 0.1
    got, plan = _csr_layer(rt, nodes, indptr, indices, w, b, mode, relu, out_bf16)
    assert plan.n_hub == 3                                            # the rows of degree 257, 5000 and 12345
    ar = torch.arange(n, device=rt.device)
    ref = _ref(x, _csr_agg(x, indptr, indices, ar, mode), w, b, relu, mode)
    if out_bf16:
        ref = ref.bfloat16().float()
    err = (got - ref).abs().max()
    assert err <= 2e-2 * ref.abs().max() + 1e-3, (float(err), float(ref.abs().max()))
    got2, _ = _csr_layer(rt, nodes, indptr, indices, w, b, mode, relu, out_bf16)
    assert torch.equal(got, got2)                                     # deterministic, hub rows included


@pytest.mark.parametrize("mode", AGGS)
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("d", [16, 100, 256])
def test_csr_layer_max_gcn_on_integers(rt, mode, dt, d):
    """{-1, 0, 1} data across round boundaries (64, 128) and hub rows (hub degree lowered to 100): max equals the oracle
    bit for bit; gcn divides by deg + 1, so it is compared within one bf16 rounding of the A tile."""
    n, n_out = 1200, 40
    g = torch.Generator(device=rt.device).manual_seed(d + 7)
    nodes, x = _table(rt, torch.randint(-1, 2, (n, d), device=rt.device, generator=g).float(), DTYPES[dt])
    deg = _degrees(n, d + 1, hi=30, special=[0, 1, 63, 64, 65, 100, 101, 127, 128, 129, 192, 200] + SPECIAL_DEGREES[-2:])
    indptr, indices = _csr(rt, deg, n, d + 1)
    w = torch.randint(-1, 2, (n_out, d if mode == "gcn" else 2 * d), device=rt.device, generator=g).float()
    b = torch.randint(-3, 4, (n_out,), device=rt.device, generator=g).float()
    got, plan = _csr_layer(rt, nodes, indptr, indices, w, b, mode, False, False, hub_degree=100)
    assert plan.n_hub == 8
    ref = _ref(x, _csr_agg(x, indptr, indices, torch.arange(n, device=rt.device), mode), w, b, False, mode)
    if mode == "max":
        assert torch.equal(got, ref), float((got - ref).abs().max())
    else:
        assert float((got - ref).abs().max()) <= 1e-2 * float(ref.abs().max()) + 1e-3


# ------------------------------------------------------------------------------- 4. engine gradients vs autograd
@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("L,fan,B,ncls", [(2, [25, 10], 512, 47), (3, [5, 4, 3], 128, 47), (3, [5, 4, 3], 128, 172)])
def test_fast_engine_agg_matches_autograd(rt, first_max_oracle, agg, L, fan, B, ncls):
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, ncls, seed=7)
    torch.manual_seed(0)
    m1 = EgoGraphSAGE(100, 256, ncls, L, agg_type=agg).to(rt.device)
    m2 = copy.deepcopy(m1)
    tr = FastSageTrainer(rt, nodes, csr, m1, fan, B, use_cuda_graph=False)
    if ncls == 172 and agg == "max":          # (gcn's K is half as wide: its 172-class W fits one image)
        assert tr.n_split[-1] > 1
    seeds = torch.randint(0, 30000, (B,), device=rt.device)
    tr.seeds.copy_(seeds)
    hops = tr.sample(seeds)
    tr.sample = lambda s: hops
    tr.opt.advance = lambda *a, **k: None
    tr._skip_opt = True                       # keep the gradients (the fused Adam kernel would zero them)
    tr._step_body()
    torch.cuda.synchronize()
    g_fast = torch.cat([p.grad.reshape(-1) for p in m1.parameters()])
    loss_fast = float(tr.loss)
    _engine_routes(first_max_oracle, tr, m2)
    logits = m2.forward_store(nodes, hops, fan)
    loss = F.cross_entropy(logits, nodes.labels.local[seeds])
    loss.backward()
    g_ref = torch.cat([p.grad.reshape(-1) for p in m2.parameters()])
    assert abs(loss_fast - float(loss)) < 2e-2 * max(1.0, abs(float(loss))), (loss_fast, float(loss))
    rel = (g_fast - g_ref).abs().max() / (g_ref.abs().max() + 1e-8)
    assert rel < 0.05, float(rel)
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("kind", ["sigmoid", "softmax"])
@pytest.mark.parametrize("L,fan", [(2, [10, 5]), (3, [5, 4, 3])])
def test_link_engine_agg_matches_autograd(rt, first_max_oracle, agg, kind, L, fan):
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    from tests.test_link_engine_gpu import _ref_loss
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, 47, seed=7)
    torch.manual_seed(0)
    m1 = EgoGraphSAGE(100, 256, 64, L, agg_type=agg).to(rt.device)
    m2 = copy.deepcopy(m1)
    B, n, T = 128, 5, (0.5 if kind == "softmax" else 1.0)
    tr = FastLinkSageTrainer(rt, nodes, csr, m1, fan, B, n, loss=kind, temperature=T, use_cuda_graph=False)
    tr.seeds[:2 * B] = torch.randint(0, 30000, (2 * B,), device=rt.device)
    tr._draw_roots(tr.seeds)
    hops = tr.sample(tr.seeds)
    tr.sample = lambda s: hops
    tr._draw_roots = lambda r: None
    tr.opt.advance = lambda *a, **k: None
    tr._skip_opt = True
    tr._step_body()
    torch.cuda.synchronize()
    g_fast = torch.cat([p.grad.reshape(-1) for p in m1.parameters()])
    loss_fast = float(tr.loss)
    _engine_routes(first_max_oracle, tr, m2)
    loss = _ref_loss(m2.forward_store(nodes, hops, fan), B, n, kind, T)
    loss.backward()
    loss = float(loss.detach())
    g_ref = torch.cat([p.grad.reshape(-1) for p in m2.parameters()])
    assert abs(loss_fast - loss) < 2e-2 * max(1.0, abs(loss)), (loss_fast, loss)
    rel = (g_fast - g_ref).abs().max() / (g_ref.abs().max() + 1e-8)
    # max hands a column's whole gradient to one child, and the temperature-0.5 softmax loss sharpens it further: the
    # bf16 rounding of H and dA (and the ReLU masks it flips) shows more in the max-abs ratio than with mean
    assert rel < (0.08 if agg == "max" else 0.05), float(rel)
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]


# ------------------------------------------------------------------------------------------------ 5. training
def _homophilous_graph(rt, n, deg, feat, n_cls, seed):
    """labelled graph whose edges stay inside a class, features = class centre * 0.5 + noise: the label is learnable from
    the neighbourhood too (gcn's mean dilutes the node's own row by 1 / (k + 1) per layer, so on a graph with random
    edges it has little left to learn from)"""
    from graphlearn_b200.store.shards import CsrShard, IdMap, NodeTable
    dev = rt.device
    g = torch.Generator(device=dev).manual_seed(seed)
    labels = torch.randint(0, n_cls, (n,), device=dev, generator=g)
    x = torch.randn(n_cls, feat, device=dev, generator=g)[labels] * 0.5 + torch.randn(n, feat, device=dev, generator=g)
    order = torch.argsort(labels)
    counts = torch.bincount(labels, minlength=n_cls)
    start = torch.cumsum(counts, 0) - counts
    src = torch.arange(n, device=dev).repeat_interleave(deg)
    c = labels[src]
    dst = order[start[c] + (torch.rand(src.numel(), device=dev, generator=g) * counts[c]).long().clamp(max=n - 1)]
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=dev), dense=True))
    nodes.set_float(x, torch.float32)
    nodes.set_labels(labels)
    return nodes, CsrShard.from_coo(rt, "e", "n", "n", src, dst, n)


@pytest.mark.parametrize("agg", AGGS)
def test_fast_engine_agg_learns_3layer(rt, agg):
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    nodes, csr = _homophilous_graph(rt, 20000, 20, 64, 8, seed=9)
    torch.manual_seed(0)
    tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 8, 3, agg_type=agg).to(rt.device), [5, 4, 3], 256, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    tr.capture()
    losses = []
    for _ in range(80):
        loss = tr.step(torch.randint(0, 20000, (256,)))
        torch.cuda.synchronize()
        losses.append(float(loss))
    assert losses[-1] < 0.6 * losses[0], (losses[0], losses[-1])


# ----------------------------------------------------------------------------------------------- 6. inference
def _oracle_forward(tr):
    """layer-wise full-neighbourhood forward in torch, with the bf16 rounding of the hidden layers"""
    from graphlearn_b200.ops import sage as S
    nodes, csr = tr.nodes, tr.csr
    h = nodes.feats.local[:, :nodes.float_dim].float()
    ar = torch.arange(h.size(0), device=h.device)
    for l, c in enumerate(tr.convs):
        last = l == len(tr.convs) - 1
        w = S.logical_weight(c.weight_p.detach(), c.in_self, c.in_nbr, c.agg_type)
        y = _ref(h, _csr_agg(h, csr.indptr.local, csr.indices.local, ar, c.agg_type), w,
                 None if c.bias is None else c.bias.detach(), not last, c.agg_type)
        h = y if last else y.bfloat16().float()
    return h


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("L,n_cls,fan", [(2, 47, [25, 10]), (3, 172, [5, 4, 3])])
def test_infer_all_agg_matches_layerwise_oracle(rt, agg, L, n_cls, fan):
    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 100, n_cls, seed=3)
    torch.manual_seed(1)
    tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, n_cls, L, agg_type=agg).to(rt.device), fan, 256,
                         use_cuda_graph=False)
    for _ in range(3):
        tr.step(torch.randint(0, 20000, (256,)))
    torch.cuda.synchronize()
    got = tr.infer_all()
    torch.cuda.synchronize()
    assert got.shape == (nodes.n_local, n_cls) and got.dtype == torch.float32
    ref = _oracle_forward(tr)
    err = (got - ref).abs().max()
    assert err <= 2e-2 * ref.abs().max(), (float(err), float(ref.abs().max()))
    assert torch.equal(got, tr.infer_all())                           # deterministic


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("link", [False, True], ids=["supervised", "link"])
def test_infer_all_agg_equals_predict_when_sampling_draws_every_neighbour(rt, agg, link):
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 5000, 50000, 64, 8, seed=5, skew=0)
    assert bool(((csr.indptr.local[1:] - csr.indptr.local[:-1]) == 10).all())
    torch.manual_seed(2)
    if link:
        tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 32, 2, agg_type=agg).to(rt.device), [10, 10], 128,
                                 3, strategy="random_without_replacement", use_cuda_graph=False)
    else:
        tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 8, 2, agg_type=agg).to(rt.device), [10, 10], 128,
                             strategy="random_without_replacement", use_cuda_graph=False)
    vids = torch.arange(0, 5000, 3, device=rt.device)
    sampled = (tr.embed(vids) if link else tr.predict(vids)).float()
    full = tr.infer_all()[vids]
    err = (sampled - full).abs().max()
    assert err <= 3e-2 * sampled.abs().max(), (float(err), float(sampled.abs().max()))


# ------------------------------------------------------------------------------------------------ 7. launches
@pytest.mark.parametrize("agg", AGGS)
def test_agg_step_launch_count(rt, agg):
    """An eager step launches 9 (supervised) / 12 (link) kernels of this repository and no library kernel, whatever the
    aggregator: the argmax bytes and the gradient routing ride in the existing launches."""
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    from tests.test_link_engine_gpu import _count_launches
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    sup = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2, agg_type=agg).to(rt.device), [25, 10], 256,
                          use_cuda_graph=False)
    sup._step_body()
    s_own, s_lib, s_names = _count_launches(sup._step_body)
    B = 128
    tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 64, 2, agg_type=agg).to(rt.device), [25, 10], B, 5,
                             use_cuda_graph=False)
    e = (torch.randint(0, 20000, (B,)), torch.randint(0, 20000, (B,)))
    tr.step(*e)
    own, lib, names = _count_launches(lambda: tr.step(*e))
    assert s_lib == 0 and lib == 0, (s_lib, lib)
    assert s_own == 9, s_names
    assert own == 12, names
