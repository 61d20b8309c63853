"""GPU numerics / semantics tests: every sm_90a kernel against a plain PyTorch
fp32 reference of the same op (run with ``pytest -m gpu`` on an H100)."""
import math
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


@pytest.fixture(scope="module")
def graph(rt):
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 5000, 60000, 100, 7, weighted=True, seed=1)
    return nodes, csr


def _adj(csr):
    ip = csr.indptr.local.cpu()
    idx = csr.indices.local.cpu()
    return ip, idx


def test_extension_loaded():
    from graphlearn_b200.parallel.runtime import native
    C = native()
    assert hasattr(C, "sage_fused_forward")


def test_sample_random_membership(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    src = torch.randint(0, 5000, (512,), device=rt.device)
    nbr, eid = S.sample_neighbors(csr, src, 25, "random")
    assert nbr.shape == (512, 25) and eid.shape == (512, 25)
    ip, idx = _adj(csr)
    nb, ei, sc = nbr.cpu(), eid.cpu(), src.cpu()
    for b in range(512):
        s, e = int(ip[sc[b]]), int(ip[sc[b] + 1])
        if e == s:
            assert (nb[b] == 0).all() and (ei[b] == -1).all()
        else:
            assert ((ei[b] >= s) & (ei[b] < e)).all()
            assert (idx[ei[b]] == nb[b]).all()


def test_sample_random_uniform(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    ip, idx = _adj(csr)
    deg = ip[1:] - ip[:-1]
    v = int(torch.argmax((deg >= 8).to(torch.int64) * (deg <= 16).to(torch.int64)))
    d = int(deg[v])
    src = torch.full((4096,), v, device=rt.device, dtype=torch.int64)
    _, eid = S.sample_neighbors(csr, src, 10, "random")
    counts = torch.bincount((eid.reshape(-1) - int(ip[v])).cpu(), minlength=d).float()
    expect = counts.sum() / d
    chi2 = float(((counts - expect) ** 2 / expect).sum())
    assert chi2 < 3 * d + 30, chi2        # very loose: df = d-1


def test_sample_without_replacement(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    src = torch.arange(0, 1000, device=rt.device)
    nbr, eid = S.sample_neighbors(csr, src, 8, "random_without_replacement")
    ip, idx = _adj(csr)
    e = eid.cpu()
    for b in range(1000):
        s, t = int(ip[b]), int(ip[b + 1])
        d = t - s
        if d == 0:
            assert (e[b] == -1).all()
            continue
        assert ((e[b] >= s) & (e[b] < t)).all()
        if d >= 8:
            assert e[b].unique().numel() == 8
        else:   # circular padding: first d distinct, then repeats
            assert e[b][:d].unique().numel() == d
            assert (e[b][d:] == e[b][: 8 - d]).all()


def test_sample_topk(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    src = torch.arange(0, 500, device=rt.device)
    nbr, eid = S.sample_neighbors(csr, src, 4, "topk")
    ip, _ = _adj(csr)
    e = eid.cpu()
    w = csr.weights.local.cpu()
    for b in range(500):
        s, t = int(ip[b]), int(ip[b + 1])
        d = t - s
        if d == 0:
            continue
        exp = torch.tensor([s + (j % d) for j in range(4)])
        assert (e[b] == exp).all()
        if d >= 2:
            assert w[s] >= w[s + 1]           # rows sorted by weight desc


def test_sample_edge_weight_distribution(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    ip, _ = _adj(csr)
    deg = ip[1:] - ip[:-1]
    v = int(torch.argmax((deg >= 6).to(torch.int64) * (deg <= 12).to(torch.int64)))
    s, d = int(ip[v]), int(deg[v])
    w = csr.weights.local[s:s + d].cpu().double()
    src = torch.full((8192,), v, device=rt.device, dtype=torch.int64)
    _, eid = S.sample_neighbors(csr, src, 8, "edge_weight")
    counts = torch.bincount((eid.reshape(-1) - s).cpu(), minlength=d).double()
    p = w / w.sum()
    expect = counts.sum() * p
    chi2 = float(((counts - expect) ** 2 / expect).sum())
    assert chi2 < 3 * d + 40, (chi2, counts, expect)


def test_sample_full_and_degree(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    src = torch.randint(0, 5000, (300,), device=rt.device)
    vals, eids, off = S.sample_full(csr, src)
    ip, idx = _adj(csr)
    sc = src.cpu()
    deg = S.get_degrees(csr, src).cpu()
    assert (deg == (ip[sc + 1] - ip[sc])).all()
    o = off.cpu()
    for b in range(300):
        s, t = int(ip[sc[b]]), int(ip[sc[b] + 1])
        assert (vals[o[b]:o[b + 1]].cpu() == idx[s:t]).all()


def test_id_filter(rt, graph):
    from graphlearn_b200.ops import sampling as S
    nodes, csr = graph
    ip, idx = _adj(csr)
    src = torch.arange(0, 400, device=rt.device)
    first = torch.tensor([int(idx[int(ip[b])]) if ip[b + 1] > ip[b] else -5 for b in range(400)], device=rt.device)
    for strat in ("random", "random_without_replacement", "topk"):
        nbr, eid = S.sample_neighbors(csr, src, 6, strat, filter_mode=S.FILTER_ID, filter_values=first)
        nb = nbr.cpu()
        for b in range(400):
            s, t = int(ip[b]), int(ip[b + 1])
            others = (idx[s:t] != first[b].cpu()).sum()
            if others > 0:
                assert (nb[b] != first[b].cpu()).all(), (strat, b)


def test_timestamp_filter_kernel(rt):
    """FILTER_TS on the kernel path: only edges with ts < bound are eligible (rows are ts-ascending), for every strategy."""
    from graphlearn_b200.ops import sampling as S
    from graphlearn_b200.store.shards import CsrShard
    g = torch.Generator(device=rt.device).manual_seed(4)
    n, E = 600, 12000
    src = torch.randint(0, n, (E,), device=rt.device, generator=g)
    dst = torch.randint(0, n, (E,), device=rt.device, generator=g)
    ts = torch.randint(0, 1000, (E,), device=rt.device, generator=g)
    csr = CsrShard.from_coo(rt, "e", "v", "v", src, dst, n, ts=ts)
    ip, idx, tsl = csr.indptr.local.cpu(), csr.indices.local.cpu(), csr.ts.local.cpu()
    q = torch.arange(0, n, device=rt.device)
    bound = torch.randint(0, 1000, (n,), device=rt.device, generator=g)
    for strat in ("random", "random_without_replacement", "topk"):
        nbr, eid = S.sample_neighbors(csr, q, 5, strat, filter_mode=S.FILTER_TS, filter_values=bound)
        nb, ei, bd = nbr.cpu(), eid.cpu(), bound.cpu()
        for b in range(n):
            a, e = int(ip[b]), int(ip[b + 1])
            ok = [(int(idx[p]), p) for p in range(a, e) if int(tsl[p]) < int(bd[b])]
            if not ok:
                assert (nb[b] == 0).all(), (strat, b)                    # default neighbour id
                continue
            allowed = {v for v, _ in ok}
            assert all(int(x) in allowed for x in nb[b]), (strat, b)
            assert all(a <= int(p) < e and int(tsl[int(p)]) < int(bd[b]) for p in ei[b] if int(p) >= 0), (strat, b)
            if strat == "random_without_replacement" and len(ok) >= 5:
                assert len(set(ei[b].tolist())) == 5, b


def test_in_degree_strategy_distribution(rt):
    """strategy 'in_degree': neighbour j of a row is drawn with probability ~ in-degree(dst_j) (chi-square)."""
    from graphlearn_b200.ops import sampling as S
    from graphlearn_b200.store.shards import CsrShard
    n = 64
    # vertex 0 points at 1..8; the in-degree of target t is made t (other sources point at it t - 1 more times)
    src, dst = [0] * 8, list(range(1, 9))
    for t in range(1, 9):
        src += [10 + i for i in range(t - 1)]
        dst += [t] * (t - 1)
    src_t, dst_t = torch.tensor(src, device=rt.device), torch.tensor(dst, device=rt.device)
    csr = CsrShard.from_coo(rt, "e", "v", "v", src_t, dst_t, n)
    indeg = torch.bincount(dst_t, minlength=n)
    csr.set_indegree_weights(indeg[csr.indices.local])
    draws = 40000
    nbr, _ = S.sample_neighbors(csr, torch.zeros(draws // 8, dtype=torch.int64, device=rt.device), 8, "in_degree")
    cnt = torch.bincount(nbr.reshape(-1).cpu(), minlength=9)[1:9].double()
    assert int(cnt.sum()) == draws
    expect = torch.arange(1, 9).double() / 36.0 * draws
    chi2 = float(((cnt - expect) ** 2 / expect).sum())
    assert chi2 < 24.3, (chi2, cnt.tolist())          # 7 d.o.f., p = 0.001


def test_node2vec_bias_distribution(rt):
    """second step of a node2vec walk on a small graph: return / common-neighbour / outward candidates are taken with
    probabilities ~ 1/p : 1 : 1/q (rejection sampling in the walk kernel)."""
    from graphlearn_b200.ops import walk as WK
    from graphlearn_b200.store.shards import CsrShard
    # 0 -> 1 ; 1 -> {0 (return), 2 (also a neighbour of 0: distance 1), 3 (distance 2)} ; 0 -> 2 as well
    edges = [(0, 1), (0, 2), (1, 0), (1, 2), (1, 3), (2, 0), (3, 1)]
    src = torch.tensor([e[0] for e in edges], device=rt.device)
    dst = torch.tensor([e[1] for e in edges], device=rt.device)
    csr = CsrShard.from_coo(rt, "e", "v", "v", src, dst, 4)
    p, q = 0.25, 4.0
    walks = WK.random_walk(csr, torch.zeros(60000, dtype=torch.int64, device=rt.device), 2, p, q).cpu()
    via1 = walks[walks[:, 0] == 1]
    assert via1.size(0) > 20000
    cnt = torch.bincount(via1[:, 1], minlength=4).double()
    w = torch.tensor([1.0 / p, 0.0, 1.0, 1.0 / q]).double()          # to 0 (return), -, to 2 (common), to 3 (outward)
    expect = w / w.sum() * via1.size(0)
    assert cnt[1] == 0
    m = expect > 0
    chi2 = float((((cnt - expect) ** 2)[m] / expect[m]).sum())
    assert chi2 < 13.8, (chi2, cnt.tolist(), expect.tolist())          # 2 d.o.f., p = 0.001


def test_gather_rows_and_agg(rt, graph):
    from graphlearn_b200.ops import gather as G
    nodes, csr = graph
    vids = torch.randint(-1, 5200, (1000,), device=rt.device)     # includes invalid ids
    out = G.gather_rows(rt, nodes.feats, nodes.feat_desc, vids, 100)
    ok = (vids >= 0) & (vids < 5000)
    ref = torch.where(ok[:, None], nodes.feats.local[vids.clamp(0, 4999), :100], torch.zeros(1, device=rt.device))
    assert torch.equal(out, ref)
    v2 = torch.randint(0, 5000, (64, 10), device=rt.device)
    for mode in ("sum", "mean", "max", "min", "prod"):
        a = G.gather_agg(rt, nodes.feats, nodes.feat_desc, v2, 100, mode, k=10)
        r = G.segment_reduce(nodes.feats.local[v2.reshape(-1), :100], mode, k=10)
        assert torch.allclose(a, r, rtol=1e-4, atol=1e-4), mode
    offs = torch.tensor([0, 3, 3, 10, 64], device=rt.device)
    flat = v2.reshape(-1)[:64]
    for mode in ("sum", "mean", "max"):
        a = G.gather_agg(rt, nodes.feats, nodes.feat_desc, flat, 100, mode, offsets=offs)
        r = G.segment_reduce(nodes.feats.local[flat, :100], mode, offsets=offs)
        assert torch.allclose(a, r, rtol=1e-4, atol=1e-4), mode


def test_gather_bf16_table(rt):
    from graphlearn_b200.store.synthetic import make_sharded_graph
    from graphlearn_b200.ops import gather as G
    nodes, csr = make_sharded_graph(rt, 3000, 20000, 100, 5, feature_dtype=torch.bfloat16, seed=3)
    vids = torch.randint(0, 3000, (777,), device=rt.device)
    out = G.gather_rows(rt, nodes.feats, nodes.feat_desc, vids, 100)
    assert torch.equal(out, nodes.feats.local[vids, :100].float())


@pytest.mark.parametrize("cfg", [
    dict(M=300, k=10, ds=100, dn=100, n_out=256, mode="mean", relu=True, bf16=True),
    dict(M=1024, k=25, ds=100, dn=100, n_out=256, mode="mean", relu=True, bf16=True),
    dict(M=129, k=5, ds=64, dn=32, n_out=47, mode="sum", relu=False, bf16=False),
    dict(M=256, k=7, ds=100, dn=100, n_out=64, mode="gcn", relu=False, bf16=False),
    dict(M=500, k=3, ds=200, dn=200, n_out=64, mode="mean", relu=True, bf16=False),
])
def test_sage_fused_store_numerics(rt, cfg):
    """wgmma fused layer reading a (fp32) store vs fp32 torch reference."""
    from graphlearn_b200.ops import sage as SG
    from graphlearn_b200.store.shards import IdMap, NodeTable
    M, k, ds, dn = cfg["M"], cfg["k"], cfg["ds"], cfg["dn"]
    n = 4000
    g = torch.Generator(device=rt.device).manual_seed(0)

    def table(d):
        t = NodeTable(rt, "t", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
        t.set_float(torch.randn(n, d, device=rt.device, generator=g))
        return t

    ts = table(ds)
    tn = ts if dn == ds else table(dn)
    sv = torch.randint(0, n, (M,), device=rt.device, generator=g)
    nv = torch.randint(0, n, (M * k,), device=rt.device, generator=g)
    kin = dn if cfg["mode"] == "gcn" else ds + dn
    w = torch.randn(cfg["n_out"], kin, device=rt.device, generator=g) / math.sqrt(kin)
    b = torch.randn(cfg["n_out"], device=rt.device, generator=g)
    assert SG.fused_supported(ds, dn, cfg["n_out"], cfg["mode"])
    y = SG.sage_layer(SG.pad_weight(w, ds, dn, cfg["mode"]), b, k=k, mode=cfg["mode"], relu=cfg["relu"], out_bf16=cfg["bf16"], self_table=ts,
                      self_vids=sv, nbr_table=tn, nbr_vids=nv).float()
    ref = SG.sage_layer_reference(w, b, ts.feats.local[sv, :ds], tn.feats.local[nv, :dn], k, cfg["mode"], cfg["relu"])
    err = (y - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err < 0.03 * max(scale, 1.0), (err, scale)


def _int_table(rt, n, d, dtype, seed):
    """Feature table with small INTEGER values: exactly representable in bf16, so the fused kernel (bf16 A
    tile, fp32 accumulation) must reproduce an fp32 reference bit for bit - a wrong-row bug cannot hide
    inside a tolerance."""
    from graphlearn_b200.store.shards import IdMap, NodeTable
    g = torch.Generator(device=rt.device).manual_seed(seed)
    t = NodeTable(rt, "t", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    t.set_float(torch.randint(-8, 9, (n, d), device=rt.device, generator=g).float(), dtype)
    return t, g


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("M,k,d,n_out", [(300, 10, 100, 256), (25600, 10, 100, 256), (1000, 25, 64, 128), (77, 3, 256, 47)])
def test_sage_fused_exact_rows(rt, M, k, d, n_out, dtype):
    """Exact-equality check of the persistent fused kernel (gather + sum + wgmma GEMM) on integer data."""
    from graphlearn_b200.ops import sage as SG
    n = 50000
    t, g = _int_table(rt, n, d, dtype, 1)
    sv = torch.randint(0, n, (M,), device=rt.device, generator=g)
    nv = torch.randint(-1, n, (M * k,), device=rt.device, generator=g)       # -1 = missing neighbour -> zero row
    w = torch.randint(-1, 2, (n_out, 2 * d), device=rt.device, generator=g).float()
    b = torch.randint(-3, 4, (n_out,), device=rt.device, generator=g).float()
    y = SG.sage_layer(SG.pad_weight(w, d, d, "sum"), b, k=k, mode="sum", relu=True, out_bf16=False, self_table=t,
                      self_vids=sv, nbr_table=t, nbr_vids=nv)
    feats = t.feats.local[:, :d].float()
    xn = torch.where((nv >= 0)[:, None], feats[nv.clamp(min=0)], torch.zeros(1, device=rt.device))
    ref = SG.sage_layer_reference(w, b, feats[sv], xn, k, "sum", True)
    torch.cuda.synchronize()
    assert torch.equal(y, ref), float((y - ref).abs().max())


@pytest.mark.parametrize("d,k,M", [(100, 10, 3000), (64, 25, 500), (37, 3, 77)])
def test_fp8_block_scaled_feature_rows(rt, d, k, M):
    """fp8 (e4m3, one bf16 scale per 32 elements) feature storage: the lookup kernel returns exactly the dequantised values and
    the fused layer equals the same layer fed with the dequantised rows."""
    from graphlearn_b200.ops import gather as G
    from graphlearn_b200.ops import sage as SG
    from graphlearn_b200.store.shards import IdMap, NodeTable
    n, n_out = 20000, 128
    g = torch.Generator(device=rt.device).manual_seed(7)
    x = torch.randn(n, d, device=rt.device, generator=g) * torch.rand(n, 1, device=rt.device, generator=g) * 4
    t8 = NodeTable(rt, "t8", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    t8.set_float(x, torch.float8_e4m3fn)
    deq = t8.dequantize_local()
    assert t8.feats.local.dtype == torch.uint8 and float(((deq - x).abs() / x.abs().amax(1, keepdim=True).clamp(min=1e-6)).max()) < 0.07
    q = torch.randint(-1, n + 5, (4000,), device=rt.device, generator=g)
    got = G.gather_rows(rt, t8.feats, t8.feat_desc, q, d)
    ok = (q >= 0) & (q < n)
    want = torch.where(ok[:, None], deq[q.clamp(0, n - 1)], torch.zeros(1, device=rt.device))
    assert torch.equal(got, want)
    # fused layer: fp8 table vs a bf16 table that stores the dequantised values (exact in bf16: 4-bit mantissa x bf16 scale)
    tb = NodeTable(rt, "tb", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    tb.set_float(deq, torch.bfloat16)
    sv = torch.randint(0, n, (M,), device=rt.device, generator=g)
    nv = torch.randint(-1, n, (M * k,), device=rt.device, generator=g)
    w = torch.randn(n_out, 2 * d, device=rt.device, generator=g) / math.sqrt(2 * d)
    b = torch.randn(n_out, device=rt.device, generator=g)
    wp = SG.pad_weight(w, d, d, "mean")
    y8 = SG.sage_layer(wp, b, k=k, mode="mean", relu=True, out_bf16=False, self_table=t8, self_vids=sv, nbr_table=t8, nbr_vids=nv)
    yb = SG.sage_layer(wp, b, k=k, mode="mean", relu=True, out_bf16=False, self_table=tb, self_vids=sv, nbr_table=tb, nbr_vids=nv)
    xn = torch.where((nv >= 0)[:, None], deq[nv.clamp(min=0)], torch.zeros(1, device=rt.device))
    ref = SG.sage_layer_reference(w, b, deq[sv], xn, k, "mean", True)
    assert (y8 - ref).abs().max() < 0.03 * max(float(ref.abs().max()), 1.0)
    # same products, same fp32 accumulation order up to the fma contraction of the dequantisation: tiny differences only
    assert (y8 - yb).abs().max() < 2e-2 * max(float(ref.abs().max()), 1.0), float((y8 - yb).abs().max())


def test_fp8_feature_rows_train(rt):
    """the hand-scheduled engine trains from an fp8 feature table (layer 1 dequantises inside the fused kernel)"""
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 16, seed=3, feature_dtype=torch.float8_e4m3fn)
    assert nodes.feats.local.dtype == torch.uint8 and nodes.feats.local.size(1) == 128
    torch.manual_seed(0)
    model = EgoGraphSAGE(100, 256, 16, 2).to(rt.device)
    tr = FastSageTrainer(rt, nodes, csr, model, [10, 5], 512, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (512,), device=rt.device))
    tr.capture()
    losses = []
    for _ in range(40):
        tr.step_device(torch.randint(0, 20000, (512,), device=rt.device))
        torch.cuda.synchronize()
        losses.append(float(tr.loss_out))
    assert all(l == l for l in losses) and sum(losses[-5:]) < 0.8 * sum(losses[:5]), losses


def test_sage_fused_multi_segment_and_ce(rt):
    """One persistent launch over two segments (k = 25 and k = 10, the flagship's layer 1) equals two single
    launches bit for bit; the fused cross-entropy epilogue matches torch."""
    from graphlearn_b200.ops import sage as SG
    from graphlearn_b200.parallel.runtime import native
    C = native()
    n, d, n_out = 30000, 100, 256
    t, g = _int_table(rt, n, d, torch.bfloat16, 2)
    segs = [(1024, 25), (25600, 10)]
    w = torch.randn(n_out, 2 * d, device=rt.device, generator=g) / math.sqrt(2 * d)
    b = torch.randn(n_out, device=rt.device, generator=g)
    wp = SG.pad_weight(w, d, d, "mean")
    img, _ = C.pack_weight_f32(wp.contiguous(), 256, False)
    svs = [torch.randint(0, n, (M,), device=rt.device, generator=g) for M, _ in segs]
    nvs = [torch.randint(0, n, (M * k,), device=rt.device, generator=g) for M, k in segs]
    rows = sum(M for M, _ in segs)
    out = torch.zeros(rows, n_out, dtype=torch.bfloat16, device=rt.device)
    asv = torch.zeros(rows, 256, dtype=torch.bfloat16, device=rt.device)
    o = [out[:1024], out[1024:]]
    a = [asv[:1024], asv[1024:]]
    C.sage_fused_multi(t.feat_desc, t.feat_desc, svs, nvs, [0, 0], [0, 0], [M for M, _ in segs], [k for _, k in segs], o, a,
                       0, img, b, 256, n_out, True, True, [], 1, 1)
    for i, (M, k) in enumerate(segs):
        y1, a1 = C.sage_fused_forward(t.feat_desc, svs[i], t.feat_desc, nvs[i], M, k, 0, img, b, 256, n_out, True, True, True)
        assert torch.equal(y1, o[i]) and torch.equal(a1, a[i]), i
        feats = t.feats.local[:, :d].float()
        ref = SG.sage_layer_reference(w, b, feats[svs[i]], feats[nvs[i]], k, "mean", True)
        err = (o[i].float() - ref).abs().max().item()
        assert err < 0.03 * max(ref.abs().max().item(), 1.0), (i, err)
        # saved A rows = [self || mean(nbrs)] in the padded K layout
        agg = feats[nvs[i]].view(M, k, d).mean(1)
        assert torch.allclose(a[i][:, :d].float(), feats[svs[i]], atol=0) and \
            torch.allclose(a[i][:, 128:128 + d].float(), agg, rtol=1e-2, atol=1e-2)
    # ---- fused CE on a top layer (n_out = 47)
    M, k, d2, ncls = 1024, 25, 256, 47
    h = torch.randn(M + M * k, d2, device=rt.device, generator=g).to(torch.bfloat16)
    w2 = torch.randn(ncls, 2 * d2, device=rt.device, generator=g) / math.sqrt(2 * d2)
    b2 = torch.randn(ncls, device=rt.device, generator=g)
    img2, _ = C.pack_weight_f32(SG.pad_weight(w2, d2, d2, "mean").contiguous(), 64, False)
    from graphlearn_b200.parallel.runtime import local_table_desc
    hd = local_table_desc(h)
    labels = torch.randint(0, ncls, (M,), device=rt.device, generator=g)
    logits = torch.zeros(M, ncls, device=rt.device)
    dl = torch.zeros(M, 64, dtype=torch.bfloat16, device=rt.device)
    scratch = torch.zeros(64, device=rt.device)
    loss, dbias = scratch[:1], scratch[1:1 + ncls]
    C.sage_fused_multi(hd, hd, [None], [None], [0], [M], [M], [k], [logits], [None], 0, img2, b2, 64, ncls, False, False,
                       [labels, None, loss, dl, dbias], 1, 1)
    ref_logits = SG.sage_layer_reference(w2, b2, h[:M], h[M:], k, "mean", False)
    assert (logits - ref_logits).abs().max() < 0.05
    lg = logits.detach().clone().requires_grad_()
    ref_loss = torch.nn.functional.cross_entropy(lg, labels)
    ref_loss.backward()
    assert abs(float(loss) - float(ref_loss)) < 1e-3 * max(1.0, float(ref_loss)), (float(loss), float(ref_loss))
    assert (dl[:, :ncls].float() - lg.grad).abs().max() < 2e-2 * lg.grad.abs().max() + 1e-6
    assert float(dl[:, ncls:].float().abs().max()) == 0.0
    assert torch.allclose(dbias, lg.grad.sum(0), rtol=1e-3, atol=1e-5)


def test_bwd_dw_wgmma(rt):
    """dW = dZ^T A on the tensor cores (MN-major wgmma operands, split-K, red.global.add) vs torch fp32;
    then the fused variant whose dZ is computed from (H, dA_next) inside the GEMM."""
    from graphlearn_b200.parallel.runtime import native
    C = native()
    g = torch.Generator(device=rt.device).manual_seed(3)
    # (a) dense dZ: integer data -> exact
    for rows, n_out, kt in [(26624, 256, 256), (1024, 47, 512), (700, 128, 128)]:
        ld = (n_out + 63) // 64 * 64
        dzp = torch.zeros(rows, ld, dtype=torch.bfloat16, device=rt.device)
        dzp[:, :n_out] = torch.randint(-2, 3, (rows, n_out), device=rt.device, generator=g).to(torch.bfloat16)
        a = torch.randint(-2, 3, (rows, kt), device=rt.device, generator=g).to(torch.bfloat16)
        ref = dzp[:, :n_out].float().t() @ a.float()
        dw = torch.zeros(n_out, kt, device=rt.device)
        C.sage_bwd_dw(dzp[:, :n_out], None, [], [], [], [], [], [], 0, None, a, dw, None, n_out)
        torch.cuda.synchronize()
        assert torch.equal(dw, ref), (rows, n_out, kt, float((dw - ref).abs().max()))
    # (b) computed dZ (2-layer flagship shapes: seeds segment takes the self half, hop-1 segment the neighbour half / k)
    B, k, d = 1024, 25, 256
    rows = B + B * k
    h = torch.randn(rows, d, device=rt.device, generator=g).to(torch.bfloat16)
    da = torch.randn(B, 2 * d, device=rt.device, generator=g).to(torch.bfloat16)
    a = torch.randn(rows, 256, device=rt.device, generator=g).to(torch.bfloat16)
    dw = torch.zeros(d, 256, device=rt.device)
    db = torch.zeros(d, device=rt.device)
    dz_out = torch.zeros(rows, d, dtype=torch.bfloat16, device=rt.device)
    C.sage_bwd_dw(None, h, [0, B], [B, rows], [da, None], [None, da], [1, k], [1.0, 1.0 / k], d, dz_out, a, dw, db, d)
    dz_ref = torch.cat([da[:, :d].float(), (da[:, d:].float() / k).repeat_interleave(k, 0)], 0) * (h.float() > 0)
    dz16 = dz_ref.to(torch.bfloat16)
    torch.cuda.synchronize()
    assert (dz_out.float() - dz16.float()).abs().max() <= 2e-2 * dz16.float().abs().max()
    ref = dz16.float().t() @ a.float()
    assert (dw - ref).abs().max() < 2e-2 * ref.abs().max(), float((dw - ref).abs().max())
    assert torch.allclose(db, dz_ref.sum(0), rtol=2e-2, atol=2e-2 * float(dz_ref.sum(0).abs().max()))


def test_sage_fused_dense_backward(rt):
    from graphlearn_b200.ops import sage as SG
    g = torch.Generator(device=rt.device).manual_seed(1)
    M, k, d, n_out = 384, 25, 256, 47
    xs = torch.randn(M, d, device=rt.device, generator=g).to(torch.bfloat16).requires_grad_()
    xn = torch.randn(M * k, d, device=rt.device, generator=g).to(torch.bfloat16).requires_grad_()
    w = (torch.randn(n_out, 2 * d, device=rt.device, generator=g) / math.sqrt(2 * d)).requires_grad_()
    b = torch.zeros(n_out, device=rt.device, requires_grad=True)
    wp = SG.pad_weight(w.detach(), d, d, "mean").requires_grad_()
    y = SG.sage_layer(wp, b, k=k, mode="mean", relu=False, x_self=xs, x_nbr=xn)
    go = torch.randn(M, n_out, device=rt.device, generator=g)
    y.backward(go)
    xs2 = xs.detach().float().requires_grad_()
    xn2 = xn.detach().float().requires_grad_()
    w2 = w.detach().clone().requires_grad_()
    b2 = b.detach().clone().requires_grad_()
    y2 = SG.sage_layer_reference(w2, b2, xs2, xn2, k, "mean", False)
    y2.backward(go)
    assert (y - y2).abs().max() < 0.05
    for a, r, name in ((SG.logical_weight(wp.grad, d, d, "mean"), w2.grad, "w"), (b.grad, b2.grad, "b"), (xs.grad.float(), xs2.grad, "xs"),
                       (xn.grad.float(), xn2.grad, "xn")):
        rel = (a - r).abs().max() / (r.abs().max() + 1e-6)
        assert rel < 0.03, (name, float(rel))


def test_flat_adam_matches_torch(rt):
    from graphlearn_b200.ops.comm import FlatAdam
    p = torch.randn(1000, device=rt.device)
    g = torch.zeros_like(p)
    p_ref = p.clone().requires_grad_()
    opt_ref = torch.optim.Adam([p_ref], lr=1e-2)
    opt = FlatAdam(p, g, lr=1e-2)
    for i in range(5):
        grad = torch.randn(1000, device=rt.device)
        g.copy_(grad)
        p_ref.grad = grad.clone()
        opt.step()
        opt_ref.step()
    assert torch.allclose(p, p_ref.detach(), rtol=1e-4, atol=1e-5)


def test_trainer_cuda_graph_learns(rt):
    from graphlearn_b200.engine.trainer import SageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 100, 8, seed=5)
    model = EgoGraphSAGE(100, 128, 8, 2).to(rt.device)
    tr = SageTrainer(rt, nodes, csr, model, [10, 5], 512, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (512,), device=rt.device))
    tr.capture()
    assert tr.graph is not None
    losses = []
    for it in range(60):
        l = tr.step(torch.randint(0, 20000, (512,)))
        torch.cuda.synchronize()
        losses.append(float(l))
    assert losses[-1] < 0.6 * losses[0], (losses[0], losses[-1])
    # fresh randomness on every replay: the device RNG offset advanced once per step
    assert int(tr.rng.state[1].item()) >= 60


@pytest.mark.parametrize("L,hidden,fan,B,ncls", [(2, 256, [25, 10], 512, 47), (3, 256, [5, 4, 3], 128, 47),
                                                 (3, 256, [5, 4, 3], 128, 172)])
def test_fast_engine_matches_autograd(rt, L, hidden, fan, B, ncls):
    """Hand-scheduled fwd/bwd (engine/fast_sage.py) vs the autograd path on identical samples."""
    import copy
    import torch.nn.functional as F
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 30000, 600000, 100, ncls, seed=7)
    torch.manual_seed(0)
    m1 = EgoGraphSAGE(100, hidden, ncls, L).to(rt.device)
    m2 = copy.deepcopy(m1)
    tr = FastSageTrainer(rt, nodes, csr, m1, fan, B, use_cuda_graph=False)
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
    logits = m2.forward_store(nodes, hops, fan)
    labels = nodes.labels.local[seeds]
    loss = F.cross_entropy(logits, labels)
    loss.backward()
    g_ref = torch.cat([p.grad.reshape(-1) for p in m2.parameters()])
    assert abs(loss_fast - float(loss)) < 2e-2 * max(1.0, abs(float(loss))), (loss_fast, float(loss))
    n = g_ref.numel()
    rel = (g_fast - g_ref).abs().max() / (g_ref.abs().max() + 1e-8)
    assert rel < 0.05, float(rel)


def test_fast_engine_learns_3layer(rt):
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 64, 8, seed=9)
    model = EgoGraphSAGE(64, 128, 8, 3).to(rt.device)
    tr = FastSageTrainer(rt, nodes, csr, model, [5, 4, 3], 256, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    tr.capture()
    losses = []
    for it in range(80):
        l = tr.step(torch.randint(0, 20000, (256,)))
        torch.cuda.synchronize()
        losses.append(float(l))
    assert losses[-1] < 0.6 * losses[0], (losses[0], losses[-1])


def test_fast_engine_e2e_pipeline_staging(rt):
    """public step(): seeds travel pinned host -> device inside the step graph one call ahead of the
    step that trains on them, the loss comes back through the pinned slot of the same call."""
    from graphlearn_b200.engine.fast_sage import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 64, 8, seed=11)
    model = EgoGraphSAGE(64, 128, 8, 2).to(rt.device)
    tr = FastSageTrainer(rt, nodes, csr, model, [5, 4], 256, lr=5e-3)
    tr.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    tr.capture()
    s = [torch.randint(0, 20000, (256,)) for _ in range(4)]
    l0 = tr.step(s[0]); torch.cuda.synchronize()
    assert torch.equal(tr._seeds_bufs[0].cpu(), s[0]) and torch.equal(tr._seeds_bufs[1].cpu(), s[0])
    l1 = tr.step(s[1]); torch.cuda.synchronize()
    assert torch.equal(tr._seeds_bufs[0].cpu(), s[1])          # prefetched for the next call
    assert float(l0) > 0 and float(l1) > 0 and l0.is_pinned() and l0.data_ptr() != l1.data_ptr()
    l2 = tr.step(s[2]); torch.cuda.synchronize()
    assert torch.equal(tr._seeds_bufs[1].cpu(), s[2]) and float(l2) > 0
    # the eager (non-graph) trainer trains on the batch of the SAME call
    tr2 = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 8, 2).to(rt.device), [5, 4], 256, use_cuda_graph=False)
    l = tr2.step(s[3]); torch.cuda.synchronize()
    assert torch.equal(tr2.seeds.cpu(), s[3]) and float(l) > 0


def test_random_walk(rt, graph):
    from graphlearn_b200.ops import walk as WK
    nodes, csr = graph
    ip, idx = _adj(csr)
    src = torch.randint(0, 5000, (256,), device=rt.device)
    for (p, q) in ((1.0, 1.0), (0.5, 2.0)):
        w = WK.random_walk(csr, src, 8, p, q).cpu()
        assert w.shape == (256, 8)
        cur = src.cpu()
        for s in range(8):
            for b in range(256):
                a, e = int(ip[cur[b]]), int(ip[cur[b] + 1])
                if e > a:
                    assert int(w[b, s]) in set(idx[a:e].tolist()), (p, q, s, b)
                else:
                    assert int(w[b, s]) == 0
            cur = w[:, s]


def test_negative_sampler_kernel(rt, graph):
    """K2: in_degree negatives are never true neighbours; the draw follows the in-degree distribution."""
    from graphlearn_b200.graph import Graph
    from graphlearn_b200.ops import negative as NEG
    from graphlearn_b200.ops import rng as R
    from graphlearn_b200.store.graph_store import GraphStore
    nodes, csr = graph
    store = GraphStore(rt)
    store.nodes["n"], store.edges["e"] = nodes, csr
    store.topology.add("e", "n", "n")
    rng = R.DeviceRng(rt, 3)
    src = torch.randint(0, 5000, (2000,), device=rt.device)
    ip, idx = _adj(csr)
    for strat in ("random", "in_degree"):
        neg = NEG.edge_negative(store, "e", src, 5, strat, None, rng=rng, salt=11)
        assert neg.shape == (2000, 5) and int(neg.min()) >= 0 and int(neg.max()) < 5000
        if strat == "in_degree":
            nc, sc = neg.cpu(), src.cpu()
            bad = 0
            for b in range(2000):
                a = set(idx[int(ip[sc[b]]):int(ip[sc[b] + 1])].tolist())
                bad += sum(1 for x in nc[b].tolist() if x in a)
            assert bad == 0, bad
            indeg = torch.bincount(csr.indices.local, minlength=5000).float().cpu()
            # size-biased draw: E[indeg | sampled] = E[d^2]/E[d] > E[d]
            sampled_mean = indeg[neg.reshape(-1).cpu()].mean()
            assert float(sampled_mean) > float(indeg.mean()) + 0.4, (float(sampled_mean), float(indeg.mean()))


@pytest.mark.parametrize("M,K,N", [(1000, 100, 47), (4096, 256, 256), (130, 512, 64), (20000, 64, 128)])
def test_tc_linear(rt, M, K, N):
    """standalone wgmma dense layer (K7) vs fp32 reference, forward and backward."""
    from graphlearn_b200.ops.linear import tc_linear
    g = torch.Generator(device=rt.device).manual_seed(M + K)
    x = torch.randn(M, K, device=rt.device, generator=g).to(torch.bfloat16).requires_grad_()
    w = (torch.randn(N, K, device=rt.device, generator=g) / math.sqrt(K)).requires_grad_()
    b = torch.randn(N, device=rt.device, generator=g).requires_grad_()
    y = tc_linear(x, w, b, relu=False)
    assert (tc_linear(x.detach(), w.detach(), b.detach(), relu=True) - torch.relu(y.detach())).abs().max() < 1e-3
    go = torch.randn(M, N, device=rt.device, generator=g)
    y.backward(go)
    x2, w2, b2 = x.detach().float().requires_grad_(), w.detach().clone().requires_grad_(), b.detach().clone().requires_grad_()
    y2 = torch.nn.functional.linear(x2, w2, b2)   # (ReLU-mask flips near 0 make gradient comparisons ill-posed)
    y2.backward(go)
    assert (y - y2).abs().max() < 0.05
    for a_, r_, name in ((w.grad, w2.grad, "w"), (b.grad, b2.grad, "b"), (x.grad.float(), x2.grad, "x")):
        rel = (a_ - r_).abs().max() / (r_.abs().max() + 1e-6)
        assert rel < 0.05, (name, float(rel))   # bf16 operands (incl. ReLU-mask flips at ~0) vs fp32 reference


def test_sharded_embedding_gpu(rt):
    from graphlearn_b200 import nn as glnn
    emb = glnn.ShardedEmbedding(rt, 1000, 32, lr=0.1)
    w0 = emb.local_weight().clone()
    ids = torch.tensor([3, 3, 10, 999], device=rt.device)
    out = emb(ids)
    assert torch.equal(out[0], w0[3])
    out.sum().backward()
    w1 = emb.local_weight()
    assert torch.allclose(w1[3], w0[3] - 0.2, atol=1e-6) and torch.allclose(w1[10], w0[10] - 0.1, atol=1e-6)
    assert torch.equal(w1[11], w0[11])


def _lazy_adam_reference(w, steps, lr, b1=0.9, b2=0.999, eps=1e-8):
    """Adam applied to the touched rows only, duplicates summed, global step for the bias correction"""
    w = w.clone().double()
    m, v = torch.zeros_like(w), torch.zeros_like(w)
    for t, (ids, g) in enumerate(steps, 1):
        uniq, inv = torch.unique(ids, return_inverse=True)
        gs = torch.zeros(uniq.numel(), w.size(1), dtype=torch.float64).index_add_(0, inv, g.double())
        m[uniq] = b1 * m[uniq] + (1 - b1) * gs
        v[uniq] = b2 * v[uniq] + (1 - b2) * gs * gs
        w[uniq] -= lr / (1 - b1 ** t) * m[uniq] / (v[uniq].sqrt() / (1 - b2 ** t) ** 0.5 + eps)
    return w.float()


def test_sharded_embedding_sparse_adam_kernel(rt):
    """K9: sparse_adam_rows_kernel (touched rows of weight + moment tables updated in place) vs a lazy-Adam reference"""
    from graphlearn_b200 import nn as glnn
    emb = glnn.ShardedEmbedding(rt, 500, 24, lr=0.01, optimizer="adam")
    w0 = emb.local_weight().clone().cpu()
    g = torch.Generator().manual_seed(2)
    steps = []
    for _ in range(6):
        ids = torch.randint(0, 500, (64,), generator=g)
        grad = torch.randn(64, 24, generator=g)
        steps.append((ids, grad))
        out = emb(ids.to(rt.device))
        out.backward(grad.to(rt.device))
    ref = _lazy_adam_reference(w0, steps, 0.01)
    assert torch.allclose(emb.local_weight().cpu(), ref, rtol=1e-4, atol=1e-6), float((emb.local_weight().cpu() - ref).abs().max())
    untouched = torch.ones(500, dtype=torch.bool)
    for ids, _ in steps:
        untouched[ids] = False
    assert torch.equal(emb.local_weight().cpu()[untouched], w0[untouched])


def test_relabel_hash_table_kernel(rt):
    """K4: first-occurrence unique + inverse + lookup vs the portable torch path."""
    from graphlearn_b200.ops.sparse import Relabel
    g = torch.Generator().manual_seed(3)
    for n, hi in ((1, 5), (1000, 50), (200000, 70000), (50000, 10 ** 12)):
        ids = torch.randint(0, hi, (n,), generator=g)
        ids[torch.rand(n, generator=g) < 0.05] = -1
        a, b = Relabel(ids.to(rt.device)), Relabel(ids)
        assert torch.equal(a.uniq.cpu(), b.uniq) and torch.equal(a.inverse.cpu(), b.inverse)
        q = torch.randint(0, hi, (4096,), generator=g)
        assert torch.equal(a.lookup(q.to(rt.device)).cpu(), b.lookup(q))
    e = Relabel(torch.zeros(0, dtype=torch.int64, device=rt.device))
    assert e.uniq.numel() == 0


@pytest.mark.parametrize("H,D", [(1, 64), (4, 8), (2, 7), (1, 1)])
def test_edge_spmm_kernels_and_grads(rt, H, D):
    """K6 sparse: fused gather x weight -> float4-atomic scatter-add, its transpose and the edge-dot backward."""
    from graphlearn_b200.ops.sparse import _spmm_torch, spmm
    g = torch.Generator().manual_seed(5)
    n_src, n_out, E = 300, 200, 5000
    x = torch.randn(n_src, H * D, generator=g)
    row, col = torch.randint(0, n_out, (E,), generator=g), torch.randint(0, n_src, (E,), generator=g)
    w = torch.rand(E, H, generator=g)
    for use_w in (True, False):
        xa = x.clone().to(rt.device).requires_grad_(True)
        wa = w.clone().to(rt.device).requires_grad_(True) if use_w else None
        xb = x.clone().requires_grad_(True)
        wb = w.clone().requires_grad_(True) if use_w else None
        oa = spmm(xa, row.to(rt.device), col.to(rt.device), wa, n_out, heads=H)
        ob = _spmm_torch(xb, row, col, wb, n_out, H)
        assert torch.allclose(oa.cpu(), ob, atol=1e-4, rtol=1e-4)
        go = torch.randn(n_out, H * D, generator=g)
        oa.backward(go.to(rt.device)); ob.backward(go)
        assert torch.allclose(xa.grad.cpu(), xb.grad, atol=1e-4, rtol=1e-4)
        if use_w:
            assert torch.allclose(wa.grad.cpu(), wb.grad, atol=1e-4, rtol=1e-4)


def test_sparse_convs_match_cpu(rt):
    import copy
    from graphlearn_b200.nn.sparse_conv import GATConv, GCNConv, SAGEConv
    g = torch.Generator().manual_seed(7)
    x = torch.randn(120, 16, generator=g)
    ei = torch.randint(0, 120, (2, 900), generator=g)
    for conv in (GCNConv(16, 8), SAGEConv(16, 8), GATConv(16, 8, num_heads=2)):
        c2 = copy.deepcopy(conv).to(rt.device)
        a, b = conv(x, ei), c2(x.to(rt.device), ei.to(rt.device))
        assert torch.allclose(a, b.cpu(), atol=1e-4, rtol=1e-3)
        a.sum().backward(); b.sum().backward()
        for p, q in zip(conv.parameters(), c2.parameters()):
            assert torch.allclose(p.grad, q.grad.cpu(), atol=1e-3, rtol=1e-3)
