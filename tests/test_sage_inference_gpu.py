"""Layer-wise full-neighbourhood inference: the CSR neighbour mode of the fused SAGE kernel (with its hub pre-pass)
against a torch oracle, bit-exact on integer data, and ``infer_all`` / ``evaluate`` of the fused trainers."""
import copy
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

DTYPES = {"fp32": torch.float32, "bf16": torch.bfloat16, "fp8": torch.float8_e4m3fn}


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


def _table(rt, x, dtype):
    """node table holding x ([n, d] fp32) in `dtype`; returns (table, the fp32 values the kernel reads)"""
    from graphlearn_b200.store.shards import IdMap, NodeTable
    n = x.size(0)
    nodes = NodeTable(rt, "n", IdMap(rt, torch.arange(n, device=rt.device), dense=True))
    nodes.set_float(x, dtype)
    if dtype == torch.float8_e4m3fn:
        vals = nodes.dequantize_local()
    else:
        vals = nodes.feats.local[:, :x.size(1)].float()
    return nodes, vals


def _csr(rt, degrees, n_vid, seed):
    g = torch.Generator(device=rt.device).manual_seed(seed)
    deg = torch.tensor(degrees, dtype=torch.int64, device=rt.device)
    indptr = torch.zeros(deg.numel() + 1, dtype=torch.int64, device=rt.device)
    indptr[1:] = torch.cumsum(deg, 0)
    indices = torch.randint(0, n_vid, (int(indptr[-1]),), device=rt.device, generator=g)
    return indptr, indices


def _agg(x, indptr, indices, mode):
    """oracle segment mean / sum over the CSR rows (float64)"""
    n = indptr.numel() - 1
    deg = indptr[1:] - indptr[:-1]
    row = torch.repeat_interleave(torch.arange(n, device=x.device), deg)
    agg = torch.zeros(n, x.size(1), dtype=torch.float64, device=x.device).index_add_(0, row, x.double()[indices])
    if mode == "mean":
        agg = agg / deg.clamp(min=1).double()[:, None]
    return agg.float()


def _layer_ref(xs, agg, w, b, relu):
    """[self || agg] rounded to bf16 (the A tile), bf16 weights, fp32 GEMM"""
    a = torch.cat([xs, agg], 1).bfloat16().float()
    y = F.linear(a, w.bfloat16().float(), b)
    return F.relu(y) if relu else y


def _images(C, w, d, N, ns):
    """weight images of a logical [n_out, 2d] weight, N-split into `ns` images of N columns"""
    from graphlearn_b200.ops import sage as S
    return S.pack_images(S.pad_weight(w, d, d, "mean"), N, ns)


def _run_layer(rt, nodes, indptr, indices, w, b, mode, relu, out_bf16, ns=1, hub_degree=None):
    from graphlearn_b200.ops import sage as S
    from graphlearn_b200.parallel.runtime import native
    C = native()
    n, d, n_real = nodes.n_local, nodes.float_dim, w.size(0)
    N = S.image_width(n_real, ns)
    img = _images(C, w, d, N, ns)
    kw = {} if hub_degree is None else {"hub_degree": hub_degree}
    plan = S.CsrPlan(indptr, indices, n, **kw)
    n_out = n_real if ns == 1 else N
    res = torch.full((n, n_real if ns == 1 else ns * N), 7.0, device=rt.device,
                     dtype=torch.bfloat16 if out_bf16 else torch.float32)
    plan.layer(nodes.feat_desc, nodes.feat_desc, torch.arange(n, device=rt.device), res[:, :n_out], mode, img, b, N,
               n_out, relu, out_bf16, ns)
    torch.cuda.synchronize()
    return res[:, :n_real].float(), plan


# round size of the CSR walk = the 64-entry pointer scratch; default hub degree 256
SPECIAL_DEGREES = [0, 1, 63, 64, 65, 128, 129, 256, 257, 5000, 12345]


def _degrees(n, seed, hi=40, special=SPECIAL_DEGREES):
    g = torch.Generator().manual_seed(seed)
    deg = torch.randint(0, hi + 1, (n,), generator=g).tolist()
    for i, s in enumerate(special):
        deg[7 * i + 3] = s
    return deg


# ------------------------------------------------------------------------------------------- 1. kernel vs oracle
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("d", [16, 100, 128, 256])
@pytest.mark.parametrize("mode", ["mean", "sum"])
def test_csr_layer_matches_oracle(rt, dt, d, mode):
    n, n_out = 2000, 47
    relu, out_bf16 = [(False, False), (True, True), (True, False), (False, True)][[16, 100, 128, 256].index(d)]
    g = torch.Generator(device=rt.device).manual_seed(d * 7 + len(mode))
    nodes, x = _table(rt, torch.randn(n, d, device=rt.device, generator=g), DTYPES[dt])
    indptr, indices = _csr(rt, _degrees(n, d), n, d)
    w = torch.randn(n_out, 2 * d, device=rt.device, generator=g) / (2 * d) ** 0.5
    b = torch.randn(n_out, device=rt.device, generator=g) * 0.1
    got, plan = _run_layer(rt, nodes, indptr, indices, w, b, mode, relu, out_bf16)
    assert plan.n_hub == 3                                            # the rows of degree 257, 5000 and 12345
    ref = _layer_ref(x, _agg(x, indptr, indices, mode), w, b, relu)
    if out_bf16:
        ref = ref.bfloat16().float()
    err = (got - ref).abs().max()
    assert err <= 2e-2 * ref.abs().max() + 1e-3, (float(err), float(ref.abs().max()))


@pytest.mark.parametrize("dt", list(DTYPES))
def test_csr_layer_multi_image(rt, dt):
    """N-split top layer (172 classes as 3 images of 64 columns in one launch)"""
    n, d, n_out = 1500, 128, 172
    g = torch.Generator(device=rt.device).manual_seed(5)
    nodes, x = _table(rt, torch.randn(n, d, device=rt.device, generator=g), DTYPES[dt])
    indptr, indices = _csr(rt, _degrees(n, 3), n, 3)
    w = torch.randn(n_out, 2 * d, device=rt.device, generator=g) / (2 * d) ** 0.5
    b = torch.randn(n_out, device=rt.device, generator=g) * 0.1
    got, _ = _run_layer(rt, nodes, indptr, indices, w, b, "mean", False, False, ns=3)
    ref = _layer_ref(x, _agg(x, indptr, indices, "mean"), w, b, False)
    assert float((got - ref).abs().max()) <= 2e-2 * float(ref.abs().max())


# ------------------------------------------------------------------------------------- 2. bit-exact on integers
@pytest.mark.parametrize("dt", ["fp32", "bf16"])
@pytest.mark.parametrize("d", [16, 100, 256])
def test_csr_layer_exact_on_integers(rt, dt, d):
    """Sum mode with features and weights in {-1, 0, 1} and degrees <= 200: every A entry is an integer that bf16
    holds exactly and the GEMM is exact in fp32, so the output must equal the oracle bit for bit - across round
    boundaries (64, 128) and for hub rows (hub degree lowered to 100)."""
    n, n_out = 1200, 40
    g = torch.Generator(device=rt.device).manual_seed(d)
    nodes, x = _table(rt, torch.randint(-1, 2, (n, d), device=rt.device, generator=g).float(), DTYPES[dt])
    deg = _degrees(n, d + 1, hi=30, special=[0, 1, 63, 64, 65, 100, 101, 127, 128, 129, 192, 200])
    indptr, indices = _csr(rt, deg, n, d + 1)
    w = torch.randint(-1, 2, (n_out, 2 * d), device=rt.device, generator=g).float()
    b = torch.randint(-3, 4, (n_out,), device=rt.device, generator=g).float()
    got, plan = _run_layer(rt, nodes, indptr, indices, w, b, "sum", False, False, hub_degree=100)
    assert plan.n_hub == 6
    ref = _layer_ref(x, _agg(x, indptr, indices, "sum"), w, b, False)
    assert torch.equal(got, ref), float((got - ref).abs().max())


# --------------------------------------------------------------------------------- 3. engine layer-wise forward
def _oracle_forward(tr):
    """the layer-wise forward in torch, with the bf16 rounding of the hidden layers"""
    from graphlearn_b200.ops import sage as S
    nodes, csr = tr.nodes, tr.csr
    h = nodes.feats.local[:, :nodes.float_dim].float()
    for l, c in enumerate(tr.convs):
        last = l == len(tr.convs) - 1
        w = S.logical_weight(c.weight_p.detach(), c.in_self, c.in_nbr, c.agg_type)
        y = _layer_ref(h, _agg(h, csr.indptr.local, csr.indices.local, c.agg_type), w,
                       None if c.bias is None else c.bias.detach(), not last)
        h = y if last else y.bfloat16().float()
    return h


@pytest.mark.parametrize("L,n_cls,fan", [(2, 47, [25, 10]), (3, 172, [5, 4, 3])])
def test_infer_all_matches_layerwise_oracle(rt, L, n_cls, fan):
    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 100, n_cls, seed=3)
    torch.manual_seed(1)
    tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, n_cls, L).to(rt.device), fan, 256, use_cuda_graph=False)
    if n_cls == 172:
        assert tr.n_split[-1] > 1
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


# ------------------------------------------------------------------------------- 4. agrees with sampled predict
@pytest.mark.parametrize("link", [False, True], ids=["supervised", "link"])
def test_infer_all_equals_predict_when_sampling_draws_every_neighbour(rt, link):
    """Every node has degree 10 and fan-outs [10, 10] without replacement draw all neighbours: the sampled forward
    is the full-neighbourhood forward up to summation order (and bf16 rounding)."""
    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 5000, 50000, 64, 8, seed=5, skew=0)
    assert bool(((csr.indptr.local[1:] - csr.indptr.local[:-1]) == 10).all())
    torch.manual_seed(2)
    if link:
        tr = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 32, 2).to(rt.device), [10, 10], 128, 3,
                                 strategy="random_without_replacement", use_cuda_graph=False)
    else:
        tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(64, 128, 8, 2).to(rt.device), [10, 10], 128,
                             strategy="random_without_replacement", use_cuda_graph=False)
    vids = torch.arange(0, 5000, 3, device=rt.device)
    sampled = (tr.embed(vids) if link else tr.predict(vids)).float()
    full = tr.infer_all()[vids]
    err = (sampled - full).abs().max()
    assert err <= 3e-2 * sampled.abs().max(), (float(err), float(sampled.abs().max()))


# ------------------------------------------------------------------------------------- 5. training is unaffected
def _training_state(tr):
    st = [tr.flat_p, tr.g_store, tr.opt.m, tr.opt.v, tr.opt.step_t, tr.rng.state, tr.loss_out] + tr.img + \
         [t for hop in tr._hops for t in hop]
    return [t.clone() for t in st] + [tr._steps]


def test_infer_all_leaves_training_state_untouched(rt):
    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=4)
    torch.manual_seed(3)
    m = EgoGraphSAGE(100, 256, 47, 2).to(rt.device)
    trs = [FastSageTrainer(rt, nodes, csr, mm, [25, 10], 256, seed=9) for mm in (m, copy.deepcopy(m))]
    for tr in trs:
        tr.capture()
        for _ in range(3):
            tr.step_device()
    torch.cuda.synchronize()
    before = _training_state(trs[0])
    trs[0].infer_all()
    acc = trs[0].evaluate(torch.arange(0, 20000, 2, device=rt.device))
    torch.cuda.synchronize()
    assert 0.0 <= acc <= 1.0
    after = _training_state(trs[0])
    for a, b in zip(before[:-1], after[:-1]):
        assert torch.equal(a, b)
    assert before[-1] == after[-1]
    # the next step of the trainer that ran inference and of its twin that did not: the same up to the order of the
    # fp32 atomics with which a step accumulates its loss and gradients
    for tr in trs:
        tr.step_device()
    torch.cuda.synchronize()
    assert torch.allclose(trs[0].loss_out, trs[1].loss_out, rtol=1e-5, atol=0)
    assert torch.allclose(trs[0].flat_p, trs[1].flat_p, rtol=0, atol=1e-6)


# ------------------------------------------------------------------------------------------------ 6. launches
def test_infer_all_launches(rt):
    from torch.profiler import ProfilerActivity, profile

    from graphlearn_b200.engine import FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 400000, 100, 47, seed=6, skew=2)
    tr = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2).to(rt.device), [25, 10], 256,
                         use_cuda_graph=False)
    tr.infer_all()
    assert tr._inf[0].n_hub > 0
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
        tr.infer_all()
        torch.cuda.synchronize()
    names, lib = {}, 0
    for ev in prof.events():
        if ev.device_type is not None and str(ev.device_type).endswith("CUDA") and ev.name and \
                not ev.name.startswith("Memcpy") and not ev.name.startswith("Memset"):
            if "glb::" in ev.name:
                key = ev.name.split("<")[0].replace("void ", "")
                names[key] = names.get(key, 0) + 1
            else:
                lib += 1
    assert lib == 0, names
    assert names == {"glb::sage_persist_kernel": 2, "glb::sage_hub_partial_kernel": 2}, names


# ---------------------------------------------------------------------------------------------- 7. two ranks
@pytest.mark.multigpu
def test_infer_all_two_ranks():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ)
    env["PYTHONPATH"] = root
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", "29683", os.path.join(root, "tests", "dist_infer_worker.py")]
    p = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    assert p.returncode == 0 and "DIST_INFER_OK" in out, out[-4000:]
