"""Unsupervised (link-prediction) GraphSAGE on the fused engine: the link loss kernel, captured negative draws, the
link trainer against autograd, its captured training, staging, edge traversal and launch count."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


def _community_graph(rt, n, deg, feat, comms, seed, p_out=0.1):
    """Graph without labels whose edges mostly stay inside a community and whose features are the community's
    centre plus noise: the link target is learnable from the features.  Returns (nodes, csr, sampler) where
    sampler(m) draws m more edges from the same process (held-out edges)."""
    from graphlearn_b200.store.shards import CsrShard, IdMap, NodeTable
    assert rt.world == 1
    dev = rt.device
    g = torch.Generator(device=dev).manual_seed(seed)
    comm = torch.randint(0, comms, (n,), device=dev, generator=g)
    centres = torch.randn(comms, feat, device=dev, generator=g)
    x = centres[comm] + 0.5 * torch.randn(n, feat, device=dev, generator=g)
    order = torch.argsort(comm)
    counts = torch.bincount(comm, minlength=comms)
    start = torch.cumsum(counts, 0) - counts

    def edges(src):
        c = comm[src]
        dst = order[start[c] + (torch.rand(src.numel(), device=dev, generator=g) * counts[c]).long().clamp(max=n - 1)]
        rnd = torch.rand(src.numel(), device=dev, generator=g) < p_out
        return torch.where(rnd, torch.randint(0, n, (src.numel(),), device=dev, generator=g), dst)

    src = torch.arange(n, device=dev).repeat_interleave(deg)
    dst = edges(src)
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=dev), dense=True))
    nodes.set_float(x, torch.float32)
    csr = CsrShard.from_coo(rt, "e", "n", "n", src, dst, n)

    def sampler(m):
        s = torch.randint(0, n, (m,), device=dev, generator=g)
        return s, edges(s)
    return nodes, csr, sampler


def _ref_loss(emb, B, n, kind, T):
    from graphlearn_b200.nn.loss import sigmoid_cross_entropy_loss, unsupervised_softmax_cross_entropy_loss
    zs, zd, zn = emb[:B], emb[B:2 * B], emb[2 * B:]
    if kind == "sigmoid":
        pos = (zs * zd).sum(-1)
        neg = (zs.unsqueeze(1) * zn.view(B, n, -1)).sum(-1).reshape(-1)
        return sigmoid_cross_entropy_loss(pos, neg)
    return unsupervised_softmax_cross_entropy_loss(zs, zd, zn, temperature=T)


# ---------------------------------------------------------------------------------------------- 1. link_loss kernel
@pytest.mark.parametrize("kind", ["sigmoid", "softmax"])
@pytest.mark.parametrize("d", [16, 64, 100, 256])
@pytest.mark.parametrize("n", [1, 5, 10])
def test_link_loss_matches_autograd(rt, kind, d, n):
    from graphlearn_b200.parallel.runtime import native
    C = native()
    B, T = 300, (0.5 if kind == "softmax" else 1.0)
    R = B * (2 + n)
    g = torch.Generator(device=rt.device).manual_seed(d * 31 + n)
    base = torch.randn(R, d + 24, device=rt.device, generator=g) * (1.5 / d ** 0.5) * 2
    emb = base[:, :d]                                            # padded rows (ld = d + 24)
    dz_buf = torch.full((R, d + 40), 7.0, device=rt.device, dtype=torch.bfloat16)
    dz = dz_buf[:, :d]
    loss = torch.zeros(4, device=rt.device)
    dbias = torch.zeros(d, device=rt.device)
    C.link_loss(emb, B, n, 0 if kind == "sigmoid" else 1, T, loss, dz, dbias)
    torch.cuda.synchronize()
    ref_emb = emb.detach().clone().requires_grad_()
    ref = _ref_loss(ref_emb, B, n, kind, T)
    ref.backward()
    gr, ref = ref_emb.grad, float(ref.detach())
    assert abs(float(loss[0]) - ref) < 1e-4 * max(1.0, abs(ref)), (float(loss[0]), ref)
    assert float(loss[1:].abs().sum()) == 0.0
    tol = 1e-2 * float(gr.abs().max()) + 1e-7                   # bf16 rounding of every row
    assert float((dz.float() - gr).abs().max()) < tol
    assert torch.all(dz_buf[:, d:] == 7.0)                       # the row padding is not written
    assert torch.allclose(dbias, gr.sum(0), rtol=1e-4, atol=1e-5 * float(gr.abs().max()) * R)


# ------------------------------------------------------------------------------------ 2. captured negative draws
def test_negative_sample_into_buffer(rt):
    from graphlearn_b200.ops import negative as NEG
    from graphlearn_b200.ops import rng as R
    from graphlearn_b200.parallel.runtime import native
    from graphlearn_b200.store.synthetic import make_sharded_graph
    C = native()
    nodes, csr = make_sharded_graph(rt, 5000, 60000, 16, 4, seed=1)
    rng = R.DeviceRng(rt, 3)
    src = torch.randint(0, 5000, (2000,), device=rt.device)
    off, total = NEG._shard_offsets(nodes, rt.device)
    indeg = torch.bincount(csr.indices.local, minlength=5000).float()
    for strict, cum in ((False, None), (True, NEG._WeightedSampler(rt, indeg).cum)):
        a = C.negative_sample(csr.desc, src, 5, cum, off, total, strict, 5, 1024, rng.state, 77, None)
        out = torch.full((2000 * 5,), -7, dtype=torch.int64, device=rt.device)
        b = C.negative_sample(csr.desc, src, 5, cum, off, total, strict, 5, 1024, rng.state, 77, out)
        assert b.data_ptr() == out.data_ptr()
        assert torch.equal(a.reshape(-1), out)


@pytest.mark.parametrize("strategy", ["random", "in_degree"])
def test_link_trainer_negatives_match_edge_negative(rt, strategy):
    """The trainer's in-place draws equal ops/negative.py::edge_negative's kernel branch for the same RNG state and
    salt (same universe, in-degree CDF and retries); in_degree negatives are never true neighbours."""
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.ops import negative as NEG
    from graphlearn_b200.store.graph_store import GraphStore
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 5000, 60000, 16, 4, seed=2)
    store = GraphStore(rt)
    store.nodes["n"], store.edges["e"] = nodes, csr
    store.topology.add("e", "n", "n")
    B, n = 400, 6
    tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(16, 32, 16, 2).to(rt.device), [4, 3], B, n,
                             neg_strategy=strategy, use_cuda_graph=False)
    src = torch.randint(0, 5000, (B,), device=rt.device)
    tr.seeds[:B] = src
    tr._draw_roots(tr.seeds)
    ref = NEG.edge_negative(store, "e", src, n, strategy, None, rng=tr.rng, salt=tr.NEG_SALT)
    torch.cuda.synchronize()
    assert torch.equal(tr.seeds[2 * B:], ref.reshape(-1))
    if strategy == "in_degree":
        ip, idx = csr.indptr.local.cpu(), csr.indices.local.cpu()
        neg, sc = ref.cpu(), src.cpu()
        for b in range(B):
            adj = set(idx[int(ip[sc[b]]):int(ip[sc[b] + 1])].tolist())
            assert not adj.intersection(neg[b].tolist()), b


# -------------------------------------------------------------------------------- 3. engine against autograd
@pytest.mark.parametrize("kind", ["sigmoid", "softmax"])
@pytest.mark.parametrize("L,fan", [(2, [10, 5]), (3, [5, 4, 3])])
def test_link_engine_matches_autograd(rt, kind, L, fan):
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, 47, seed=7)
    torch.manual_seed(0)
    m1 = EgoGraphSAGE(100, 256, 64, L).to(rt.device)
    m2 = copy.deepcopy(m1)
    B, n, T = 128, 5, (0.5 if kind == "softmax" else 1.0)
    tr = FastLinkSageTrainer(rt, nodes, csr, m1, fan, B, n, loss=kind, temperature=T, use_cuda_graph=False)
    tr.seeds[:2 * B] = torch.randint(0, 30000, (2 * B,), device=rt.device)
    tr._draw_roots(tr.seeds)
    hops = tr.sample(tr.seeds)
    tr.sample = lambda s: hops
    tr._draw_roots = lambda r: None
    tr.opt.advance = lambda *a, **k: None
    tr._skip_opt = True                       # keep the gradients (the fused Adam kernel would zero them)
    tr._step_body()
    torch.cuda.synchronize()
    g_fast = torch.cat([p.grad.reshape(-1) for p in m1.parameters()])
    loss_fast = float(tr.loss)
    emb = m2.forward_store(nodes, hops, fan)
    loss = _ref_loss(emb, B, n, kind, T)
    loss.backward()
    loss = float(loss.detach())
    g_ref = torch.cat([p.grad.reshape(-1) for p in m2.parameters()])
    assert abs(loss_fast - loss) < 2e-2 * max(1.0, abs(loss)), (loss_fast, loss)
    rel = (g_fast - g_ref).abs().max() / (g_ref.abs().max() + 1e-8)
    assert rel < 0.05, float(rel)


# ------------------------------------------------------------------------------------ 4. captured training learns
def test_link_engine_learns_captured(rt):
    from graphlearn_b200 import errors
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    nodes, csr, held_out = _community_graph(rt, n=20000, deg=12, feat=64, comms=50, seed=3)
    torch.manual_seed(0)
    model = EgoGraphSAGE(64, 128, 64, 2).to(rt.device)
    tr = FastLinkSageTrainer(rt, nodes, csr, model, [10, 5], 256, 5, lr=5e-3)
    tr.capture()
    assert tr.graph is not None
    losses = []
    while len(losses) < 80:
        try:
            l = tr.step_edges()
        except errors.OutOfRangeError:
            continue
        torch.cuda.synchronize()
        losses.append(float(l))
    assert losses[-1] < 0.6 * losses[0], (losses[0], losses[-1])
    s, d = held_out(4000)
    r = torch.randint(0, 20000, (2, 4000), device=rt.device)
    zs, zd, za, zb = (tr.embed(v) for v in (s, d, r[0], r[1]))
    pos, neg = (zs * zd).sum(-1), (za * zb).sum(-1)
    # AUC: probability that a held-out edge outscores a random pair
    auc = float((pos[:, None] > neg[None, :]).float().mean())
    assert auc > 0.75, auc


# -------------------------------------------------------------------------------------------- 5. pinned staging
def test_link_engine_e2e_pipeline_staging(rt):
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 64, 8, seed=11)
    B = 128
    tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 32, 2).to(rt.device), [5, 4], B, 3, lr=5e-3)
    tr.capture()
    e = [(torch.randint(0, 20000, (B,)), torch.randint(0, 20000, (B,))) for _ in range(4)]

    def roots(buf):
        return buf[:2 * B].cpu()
    l0 = tr.step(*e[0]); torch.cuda.synchronize()
    want0 = torch.cat(e[0])
    assert torch.equal(roots(tr._seeds_bufs[0]), want0) and torch.equal(roots(tr._seeds_bufs[1]), want0)
    l1 = tr.step(*e[1]); torch.cuda.synchronize()
    assert torch.equal(roots(tr._seeds_bufs[0]), torch.cat(e[1]))          # prefetched for the next call
    assert float(l0) > 0 and float(l1) > 0 and l0.is_pinned() and l0.data_ptr() != l1.data_ptr()
    l2 = tr.step(*e[2]); torch.cuda.synchronize()
    assert torch.equal(roots(tr._seeds_bufs[1]), torch.cat(e[2])) and float(l2) > 0
    # the eager (non-graph) trainer trains on the edges of the SAME call
    tr2 = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 32, 2).to(rt.device), [5, 4], B, 3,
                              use_cuda_graph=False)
    l = tr2.step(*e[3]); torch.cuda.synchronize()
    assert torch.equal(roots(tr2.seeds), torch.cat(e[3])) and float(l) > 0


@pytest.mark.parametrize("link", [False, True], ids=["supervised", "link"])
def test_eager_step_trains_on_its_own_batch_when_host_runs_ahead(rt, link):
    """Without CUDA graphs, step() refills pinned staging memory on the host.  When the host runs ahead of the GPU,
    a later call must not overwrite a batch that the device has not read yet: step t trains on the roots of call t."""
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 64, 8, seed=11)
    B = 128
    if link:
        tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 32, 2).to(rt.device), [5, 4], B, 3,
                                 use_cuda_graph=False)
        batches = [(torch.randint(0, 20000, (B,)), torch.randint(0, 20000, (B,))) for _ in range(4)]
    else:
        tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 8, 2).to(rt.device), [5, 4], B,
                             use_cuda_graph=False)
        batches = [(torch.randint(0, 20000, (B,)),) for _ in range(4)]
    tr.step(*batches[0]); torch.cuda.synchronize()        # first launches load their modules
    want = [torch.cat(b) for b in batches[1:3]]
    snaps = [torch.empty_like(w, device=rt.device) for w in want]
    torch.cuda._sleep(400_000_000)                         # ~0.2 s at 1.98 GHz: the GPU lags the host
    for b, snap in zip(batches[1:3], snaps):
        tr.step(*b)
        snap.copy_(tr.seeds[:snap.numel()])                # the roots this step trained on
    tr.step(*batches[3])                                   # reuses the staging memory of batches[1]
    torch.cuda.synchronize()
    for snap, w in zip(snaps, want):
        assert torch.equal(snap.cpu(), w)


# ------------------------------------------------------------------------------------- 6. edge traversal epochs
def test_link_engine_step_edges_epochs(rt):
    from graphlearn_b200 import errors
    from graphlearn_b200.engine import FastLinkSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    nodes, csr, _ = _community_graph(rt, n=2000, deg=8, feat=16, comms=10, seed=4)
    n_edges = 2000 * 8
    src_all = csr._row_of_edge.cpu()
    key_all = torch.sort(src_all * 2000 + csr.indices.local.cpu())[0]
    for B in (500, 600):                       # 16000 = 32 x 500;  26 x 600 + 400 left over
        tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(16, 32, 16, 2).to(rt.device), [3, 2], B, 2,
                                 use_cuda_graph=False)
        seen, firsts = [], []
        for epoch in range(2):
            keys = []
            while True:
                try:
                    tr.step_edges()
                except errors.OutOfRangeError:
                    break
                r = tr.seeds[:2 * B].cpu()
                keys.append(r[:B] * 2000 + r[B:])
            assert len(keys) == n_edges // B and tr.epoch == epoch + 1
            firsts.append(keys[0])
            seen.append(torch.sort(torch.cat(keys))[0])
        if n_edges % B == 0:
            assert torch.equal(seen[0], key_all) and torch.equal(seen[1], key_all)      # every edge exactly once
        else:
            for s in seen:                     # full batches of distinct edges, the remainder dropped
                assert s.numel() == (n_edges // B) * B
                assert torch.all(torch.isin(s, key_all))
        assert not torch.equal(firsts[0], firsts[1])                              # a fresh permutation per epoch


# ------------------------------------------------------------------------------------------------ 7. launches
def _count_launches(fn):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        fn()
        torch.cuda.synchronize()
    own, lib, names = 0, 0, {}
    for ev in prof.events():
        if ev.device_type is not None and str(ev.device_type).endswith("CUDA") and ev.name and \
                not ev.name.startswith("Memcpy") and not ev.name.startswith("Memset"):
            if "glb::" in ev.name:
                own += 1
                key = ev.name.split("(")[0].replace("void ", "")
                names[key] = names.get(key, 0) + 1
            else:
                lib += 1
    return own, lib, names


def test_link_engine_launch_count(rt):
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    sup = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2).to(rt.device), [25, 10], 256,
                          use_cuda_graph=False)
    sup._step_body()
    s_own, s_lib, _ = _count_launches(sup._step_body)
    B = 128
    tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 64, 2).to(rt.device), [25, 10], B, 5,
                             use_cuda_graph=False)
    e = (torch.randint(0, 20000, (B,)), torch.randint(0, 20000, (B,)))
    tr.step(*e)
    own, lib, names = _count_launches(lambda: tr.step(*e))
    assert s_lib == 0 and lib == 0, (s_lib, lib)
    for k in ("glb::link_roots_kernel", "glb::negative_sample_kernel", "glb::link_loss_kernel"):
        assert names.get(k) == 1, names
    assert own == s_own + 3, (own, s_own, names)
