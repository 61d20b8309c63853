"""Dropout between the layers of the fused GraphSAGE trainers: the forward epilogue's mask against an independent host
Philox4x32-10 of the documented mask function, bit for bit; its rate and freshness per step; the gradients of the
supervised and link trainers against autograd through the engine's mask; captured training; and the paths that never
drop (inference, launch counts, checkpoints, the rate checks)."""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_sage_agg_gpu import _engine_routes, _homophilous_graph, first_max_oracle  # noqa: F401  (fixture)
from tests.test_sage_agg_gpu import _oracle_forward as _oracle_max_gcn
from tests.test_sage_inference_gpu import _oracle_forward as _oracle_mean_sum

pytestmark = pytest.mark.gpu

AGGS = ["mean", "sum", "max", "gcn"]


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


# ------------------------------------------------------------------------------------------- host mask function
_M32 = np.uint64(0xFFFFFFFF)


def _philox4x32_10(key, c0, c1, c2, c3):
    """Philox4x32-10 (Salmon et al., SC'11) in numpy: 64-bit key, four 32-bit counter words -> four 32-bit words"""
    k0, k1 = np.uint64(key & 0xFFFFFFFF), np.uint64((key >> 32) & 0xFFFFFFFF)
    c0, c1, c2, c3 = [x.copy() for x in np.broadcast_arrays(*[np.asarray(x, dtype=np.uint64) & _M32 for x in (c0, c1, c2, c3)])]
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _M32
        k0 = (k0 + np.uint64(0x9E3779B9)) & _M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & _M32
    return c0, c1, c2, c3


def _host_keep(seed, counter, layer, rows, cols, p):
    """keep mask [rows, cols] of a layer's output buffer: element (r, c) takes the 16 bits (c % 2) of word (c / 8) % 4
    of Philox(key = seed; counter = (r, layer << 24 | (c / 32) * 4 + (c / 2) % 4, counter low, counter high)) and is
    kept when they are >= round(p * 65536).  One Philox call per (row, counter group), as the kernel draws them."""
    ngrp = (cols + 31) // 32 * 4
    r = np.arange(rows, dtype=np.uint64)[:, None]
    grp = (np.uint64(layer) << np.uint64(24)) | np.arange(ngrp, dtype=np.uint64)[None, :]
    w = np.stack(_philox4x32_10(int(seed), r, grp, counter & 0xFFFFFFFF, counter >> 32))      # [4, rows, ngrp]
    c = np.arange(cols)
    word = w[(c >> 3) & 3, :, (c >> 5) * 4 + ((c >> 1) & 3)]                                  # [cols, rows]
    bits = (word.T >> (np.uint64(16) * (c & 1).astype(np.uint64))) & np.uint64(0xFFFF)
    return torch.from_numpy(bits >= np.uint64(round(p * 65536)))


def test_host_philox_known_answers():
    """the host generator is Philox4x32-10: the Random123 known-answer vectors"""
    got = [[int(x) for x in _philox4x32_10(k, *c)] for k, c in [
        (0, (0, 0, 0, 0)),
        (0xFFFFFFFFFFFFFFFF, (0xFFFFFFFF,) * 4),
        (0xA4093822 | (0x299F31D0 << 32), (0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344))]]
    assert got == [[0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8], [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD],
                   [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]]


# ----------------------------------------------------------------------------------------------------- helpers
def _trainer(rt, nodes, csr, L, agg, p, fan, B, ncls=47, hidden=256, init_seed=0, **kw):
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    torch.manual_seed(init_seed)
    m = EgoGraphSAGE(nodes.float_dim, hidden, ncls, L, agg_type=agg, dropout=p).to(rt.device)
    return FastSageTrainer(rt, nodes, csr, m, fan, B, **kw)


def _fix_hops(tr, hops):
    """train on `hops` only, and keep the gradients and the weights (no optimiser, no counters)"""
    tr.sample = lambda s: hops
    tr.opt.advance = lambda *a, **k: None
    tr._skip_opt = True


def _undropped(tr, ly, hops):
    """layer `ly`'s forward launch again on the inputs it just read, with dropout off: its output before the mask"""
    out = torch.zeros_like(ly.Hp)
    self_base, nbr_base, Ms, ks, _, _ = ly.fwd
    outs = [out[ly.offs[i]:ly.offs[i + 1], :ly.n_out] for i in range(ly.nseg)]
    if ly.below is None:
        d, s_ids, n_ids = tr.nodes.feat_desc, hops[:ly.nseg], hops[1:ly.nseg + 1]
    else:
        d, s_ids, n_ids = ly.below, [None] * ly.nseg, [None] * ly.nseg
    tr.C.sage_fused_multi(d, d, s_ids, n_ids, self_base, nbr_base, Ms, ks, outs, [None] * ly.nseg, ly.mode, ly.img,
                          ly.conv.bias, ly.N, ly.n_out, True, True, [], 1, ly.ns, [])
    torch.cuda.synchronize()
    return out[:, :ly.conv.out_dim]


def _check_mask(tr, hops, p):
    """every hidden layer's output is nonzero exactly where its undropped output is and the host mask at the trainer's
    current counter keeps; for p = 0.5 it equals where(mask, 2 H_0, 0) bit for bit (scaling by 2 commutes with the bf16
    rounding, 1 / (1 - p) in general does not).  Returns the per-layer (kept, positive) counts."""
    seed, ctr = (int(x) for x in tr.drop_state.cpu())
    counts = []
    for l, ly in enumerate(tr.layers[:-1], 1):
        h0 = _undropped(tr, ly, hops)
        keep = _host_keep(seed, ctr, l, ly.rows, ly.conv.out_dim, p).to(h0.device)
        assert torch.equal(ly.H != 0, keep & (h0 != 0)), l
        if p == 0.5:
            want = torch.where(keep, h0 * 2, torch.zeros_like(h0))
            assert torch.equal(ly.H, want), (l, int((ly.H != want).sum()))
        counts.append((int((ly.H > 0).sum()), int((h0 > 0).sum())))
    return counts


# ------------------------------------------------------------------------------------------------ 1. exact mask
@pytest.mark.parametrize("agg", ["mean", "max"])
@pytest.mark.parametrize("L,fan,B", [(2, [25, 10], 512), (3, [5, 4, 3], 128)])
def test_dropout_mask_is_exact(rt, agg, L, fan, B):
    """p = 0.5: H_p = where(mask, 2 H_0, 0) bit for bit, against the p = 0 trainer (layer 1) and against the layer's
    own launch with dropout off (every hidden layer).  The 3-layer model's second layer (K = 512, 256 outputs) is
    N-split over four images, whose columns take the same mask as an unsplit layer's."""
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, 47, seed=7)
    trp = _trainer(rt, nodes, csr, L, agg, 0.5, fan, B, use_cuda_graph=False)
    tr0 = _trainer(rt, nodes, csr, L, agg, 0.0, fan, B, use_cuda_graph=False)
    if L == 3:
        assert trp.layers[1].ns > 1
    seeds = torch.randint(0, 30000, (B,), device=rt.device)
    trp.seeds.copy_(seeds)
    hops = trp.sample(seeds)
    for tr in (trp, tr0):
        _fix_hops(tr, hops)
        tr._step_body()
    torch.cuda.synchronize()
    _check_mask(trp, hops, 0.5)
    keep = _host_keep(*(int(x) for x in trp.drop_state.cpu()), 1, trp.layers[0].rows, trp.layers[0].conv.out_dim, 0.5)
    h0 = tr0.layers[0].H
    assert torch.equal(trp.layers[0].H, torch.where(keep.to(h0.device), h0 * 2, torch.zeros_like(h0)))


# ------------------------------------------------------------------------------------------ 2. rate, freshness
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_rate(rt, p):
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, 47, seed=7)
    tr = _trainer(rt, nodes, csr, 2, "mean", p, [25, 10], 512, use_cuda_graph=False)
    seeds = torch.randint(0, 30000, (512,), device=rt.device)
    hops = tr.sample(seeds)
    _fix_hops(tr, hops)
    tr._step_body()
    torch.cuda.synchronize()
    (kept, pos), = _check_mask(tr, hops, p)
    sigma = (pos * p * (1 - p)) ** 0.5
    assert pos > 100000 and abs(kept - pos * (1 - p)) < 5 * sigma, (kept, pos, p)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_host_masks_of_consecutive_steps_differ(p):
    a = _host_keep(12345, 7, 1, 2000, 256, p)
    b = _host_keep(12345, 8, 1, 2000, 256, p)
    agree = float((a == b).float().mean())
    assert abs(agree - (p * p + (1 - p) ** 2)) < 0.01, agree
    assert abs(float(a.float().mean()) - (1 - p)) < 0.01


def test_dropout_counter_advances_once_per_step(rt):
    """eager steps and captured replays each advance the counter by one; after them the masks are still exact at the
    current counter value"""
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    tr = _trainer(rt, nodes, csr, 2, "mean", 0.5, [25, 10], 256)
    ctr = lambda: int(tr.drop_state[1])                                 # noqa: E731
    assert ctr() == 0
    tr.step(torch.randint(0, 20000, (256,)))
    torch.cuda.synchronize()
    assert ctr() == 1                                                   # eager
    tr.capture(warmup=3)
    torch.cuda.synchronize()
    assert ctr() == 4                                                   # + 3 eager warm-up steps
    for i in range(5):
        tr.step(torch.randint(0, 20000, (256,)))
    torch.cuda.synchronize()
    assert ctr() == 9                                                   # + 5 replays
    for i in range(3):
        tr.step_device()
    torch.cuda.synchronize()
    assert ctr() == 12
    seeds = torch.randint(0, 20000, (256,), device=rt.device)
    hops = tr.sample(seeds)
    _fix_hops(tr, hops)
    tr._step_body()
    torch.cuda.synchronize()
    _check_mask(tr, hops, 0.5)
    assert ctr() == 12


# ------------------------------------------------------------------------------------------------ 3. gradients
def _check_grads(m_fast, m_ref, max_tol):
    """Every parameter's gradient within 5 % of the oracle's in norm, and the largest difference of any gradient entry
    within `max_tol` of the largest oracle entry.  The bf16 hidden activations and dA rows give the engine a relative
    error of about 3 % per parameter in norm with or without dropout (3-layer, 172 classes, mean: 0.029 at p = 0.5,
    0.029 at p = 0), but dropout halves the terms each entry sums, so the largest single-entry difference grows: 0.076 of
    the largest entry there, against the 0.05 the dropout-free tests allow."""
    errs = []
    for (name, a), b in zip(m_fast.named_parameters(), m_ref.parameters()):
        errs.append((float((a.grad - b.grad).norm() / (b.grad.norm() + 1e-12)), name))
    assert max(errs)[0] < 0.05, max(errs)
    g_fast = torch.cat([q.grad.reshape(-1) for q in m_fast.parameters()])
    g_ref = torch.cat([q.grad.reshape(-1) for q in m_ref.parameters()])
    rel = (g_fast - g_ref).abs().max() / (g_ref.abs().max() + 1e-8)
    assert rel < max_tol, float(rel)


def _oracle_logits(model, nodes, hops, fan, tr, p):
    """EgoGNN in torch: every hidden hop tensor times the engine's mask (H_p != 0) / (1 - p), once for both of its
    consumers; elements ReLU already zeroed get no gradient either way"""
    L = model.num_layers
    h = [model.convs[0].forward_store(nodes, hops[i], hops[i + 1], fan[i], relu=True, out_bf16=True) for i in range(L)]
    for l in range(1, L):
        ly = tr.layers[l - 1]
        h = [h[i] * ((ly.H[ly.offs[i]:ly.offs[i + 1]] != 0).to(h[i].dtype) / (1 - p)) for i in range(len(h))]
        last = l == L - 1
        h = [model.convs[l](h[i], h[i + 1], fan[i], relu=not last, out_bf16=not last) for i in range(L - l)]
    return h[0].float()


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("L,fan,B,ncls", [(2, [25, 10], 512, 47), (3, [5, 4, 3], 128, 47), (3, [5, 4, 3], 128, 172)])
def test_dropout_gradients_match_autograd(rt, first_max_oracle, agg, L, fan, B, ncls):  # noqa: F811
    from graphlearn_b200.store.synthetic import make_sharded_graph
    p = 0.5
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, ncls, seed=7)
    tr = _trainer(rt, nodes, csr, L, agg, p, fan, B, ncls=ncls, use_cuda_graph=False)
    m2 = copy.deepcopy(tr.model)
    seeds = torch.randint(0, 30000, (B,), device=rt.device)
    tr.seeds.copy_(seeds)
    hops = tr.sample(seeds)
    _fix_hops(tr, hops)
    tr._step_body()
    torch.cuda.synchronize()
    loss_fast = float(tr.loss)
    _engine_routes(first_max_oracle, tr, m2)
    loss = F.cross_entropy(_oracle_logits(m2, nodes, hops, fan, tr, p), nodes.labels.local[seeds])
    loss.backward()
    loss = float(loss.detach())
    assert abs(loss_fast - loss) < 2e-2 * max(1.0, abs(loss)), (loss_fast, loss)
    _check_grads(tr.model, m2, 0.1)
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]


@pytest.mark.parametrize("agg", AGGS)
@pytest.mark.parametrize("kind", ["sigmoid", "softmax"])
@pytest.mark.parametrize("L,fan", [(2, [10, 5]), (3, [5, 4, 3])])
def test_link_dropout_gradients_match_autograd(rt, first_max_oracle, agg, kind, L, fan):  # noqa: F811
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    from tests.test_link_engine_gpu import _ref_loss
    p = 0.5
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, 47, seed=7)
    torch.manual_seed(0)
    m1 = EgoGraphSAGE(100, 256, 64, L, agg_type=agg, dropout=p).to(rt.device)
    m2 = copy.deepcopy(m1)
    B, n, T = 128, 5, (0.5 if kind == "softmax" else 1.0)
    tr = FastLinkSageTrainer(rt, nodes, csr, m1, fan, B, n, loss=kind, temperature=T, use_cuda_graph=False)
    tr.seeds[:2 * B] = torch.randint(0, 30000, (2 * B,), device=rt.device)
    tr._draw_roots(tr.seeds)
    hops = tr.sample(tr.seeds)
    _fix_hops(tr, hops)
    tr._draw_roots = lambda r: None
    tr._step_body()
    torch.cuda.synchronize()
    assert bool((tr.layers[-1].H != 0).all())                         # the embeddings are never dropped
    loss_fast = float(tr.loss)
    _engine_routes(first_max_oracle, tr, m2)
    loss = _ref_loss(_oracle_logits(m2, nodes, hops, fan, tr, p), B, n, kind, T)
    loss.backward()
    loss = float(loss.detach())
    assert abs(loss_fast - loss) < 2e-2 * max(1.0, abs(loss)), (loss_fast, loss)
    _check_grads(m1, m2, 0.12 if agg == "max" else 0.1)
    assert all(a > 0.95 for a in first_max_oracle["agree"]), first_max_oracle["agree"]


# ------------------------------------------------------------------------------------------------- 4. training
@pytest.mark.parametrize("agg", AGGS)
def test_dropout_training_learns_3layer(rt, agg):
    nodes, csr = _homophilous_graph(rt, 20000, 20, 64, 8, seed=9)
    tr = _trainer(rt, nodes, csr, 3, agg, 0.5, [5, 4, 3], 256, ncls=8, hidden=128, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    tr.capture()
    losses = []
    for _ in range(80):
        loss = tr.step(torch.randint(0, 20000, (256,)))
        torch.cuda.synchronize()
        losses.append(float(loss))
    assert all(x == x for x in losses)
    # (dropout makes single steps noisy: compare the mean of the last five)
    assert sum(losses[-5:]) / 5 < 0.6 * losses[0], (losses[0], losses[-5:])


# ------------------------------------------------------------------------------------------- 5. unchanged paths
def test_dropout_step_launch_count(rt):
    """dropout rides in the existing launches: a step with p = 0.5 launches the same kernels as the step without
    dropout (9 supervised / 12 link, as tests/test_link_engine_gpu.py and test_sage_agg_gpu.py count them), only
    the forward of the hidden layer is its dropout instantiation, and no library kernel runs.  The two steps are
    profiled side by side: late in a long session the profiler was seen to report one kernel fewer for a step (8 for
    the supervised one) than the same test counts alone."""
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    from tests.test_link_engine_gpu import _count_launches
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    B = 128
    e = (torch.randint(0, 20000, (B,)), torch.randint(0, 20000, (B,)))
    counts = {}
    for p in (0.0, 0.5):
        sup = _trainer(rt, nodes, csr, 2, "mean", p, [25, 10], 256, use_cuda_graph=False)
        sup._step_body()
        tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 64, 2, dropout=p).to(rt.device), [25, 10], B, 5,
                                 use_cuda_graph=False)
        tr.step(*e)
        counts[p] = (_count_launches(sup._step_body), _count_launches(lambda: tr.step(*e)))
    for (own0, lib0, names0), (own, lib, names) in zip(counts[0.0], counts[0.5]):
        assert lib0 == 0 and lib == 0, (lib0, lib)
        assert own == own0, (names0, names)
        assert sum(v for k, v in names.items() if k.endswith(", true>")) == 1, names         # the hidden layer only
        assert {k.replace(", true>", ", false>"): v for k, v in names.items()} == names0, (names0, names)


@pytest.mark.parametrize("agg", ["mean", "max"])
def test_infer_all_never_drops(rt, agg):
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 100, 47, seed=3)
    tr = _trainer(rt, nodes, csr, 2, agg, 0.5, [25, 10], 256, init_seed=1, use_cuda_graph=False)
    for _ in range(3):
        tr.step(torch.randint(0, 20000, (256,)))
    torch.cuda.synchronize()
    got = tr.infer_all()
    torch.cuda.synchronize()
    ref = (_oracle_mean_sum if agg == "mean" else _oracle_max_gcn)(tr)
    err = (got - ref).abs().max()
    assert err <= 2e-2 * ref.abs().max(), (float(err), float(ref.abs().max()))
    assert torch.equal(got, tr.infer_all())


def test_checkpoint_carries_the_dropout_counter(rt):
    """a fresh trainer (other seed) that loads a state dict draws the original trainer's next masks; a state dict
    without the dropout state still loads"""
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    tr = _trainer(rt, nodes, csr, 2, "mean", 0.5, [25, 10], 256, use_cuda_graph=False)
    for _ in range(3):
        tr.step(torch.randint(0, 20000, (256,)))
    torch.cuda.synchronize()
    sd = tr.state_dict()
    tr2 = _trainer(rt, nodes, csr, 2, "mean", 0.5, [25, 10], 256, init_seed=5, seed=3, use_cuda_graph=False)
    assert not torch.equal(tr2.drop_state, tr.drop_state)
    tr2.load_state_dict(sd)
    assert torch.equal(tr2.drop_state, tr.drop_state) and int(tr2.drop_state[1]) == 3
    tr.repack()
    hops = tr.sample(torch.randint(0, 20000, (256,), device=rt.device))
    for t in (tr, tr2):
        _fix_hops(t, hops)
        t._step_body()
    torch.cuda.synchronize()
    assert torch.equal(tr.layers[0].H, tr2.layers[0].H)
    old = {k: v for k, v in sd.items() if k != "dropout_state"}
    tr3 = _trainer(rt, nodes, csr, 2, "mean", 0.5, [25, 10], 256, use_cuda_graph=False)
    before = tr3.drop_state.clone()
    tr3.load_state_dict(old)
    assert torch.equal(tr3.drop_state, before)


@pytest.mark.parametrize("p", [1.0, 1.5, -0.1])
def test_dropout_rate_out_of_range_raises(rt, p):
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 2000, 20000, 100, 47, seed=0)
    with pytest.raises(ValueError):
        _trainer(rt, nodes, csr, 2, "mean", p, [25, 10], 64, use_cuda_graph=False)
