"""dA = dZ . W of every layer l >= 2 on the mma.sync kernel (sage_bwd_da) over the layer's forward weight images,
against an fp32 reference, and the trainers' use of it."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    from graphlearn_b200.parallel.runtime import init
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return init()


def _within_ulp(x_bf16, ref):
    """every element of the bf16 tensor is within one bf16 ulp of the reference (plus fp32 summation noise)"""
    x, ref = x_bf16.float(), ref.float()
    tol = ref.abs() * 2.0 ** -7 + 1e-6 * ref.abs().max().item() + 1e-30
    bad = (x - ref).abs() > tol
    assert not bad.any(), ((x - ref).abs()[bad][:8], ref[bad][:8], int(bad.sum()))


@pytest.mark.parametrize("rows,n_out,kt,n_imgs,N", [
    (1024, 47, 512, 1, 64), (3584, 64, 512, 1, 64), (1000, 20, 256, 1, 64), (37, 64, 256, 1, 64),
    (16384, 256, 512, 4, 64),       # sage3's middle layer: N-split into 4 images, many row blocks per CTA
    (1024, 172, 512, 3, 64),        # sage3's top layer: 3 images, zero rows beyond 172
    (1000, 128, 256, 1, 128),       # one 128-column image
    (20037, 172, 512, 3, 64),       # row blocks per CTA with a partial last block
])
def test_sage_bwd_da_matches_fp32(rt, rows, n_out, kt, n_imgs, N):
    from graphlearn_b200.parallel.runtime import native
    C = native()
    g = torch.Generator(device=rt.device).manual_seed(rows + n_out)
    R = n_imgs * N
    w = torch.randn(n_out, kt, device=rt.device, generator=g) / math.sqrt(kt)
    dzp = torch.zeros(rows, R, dtype=torch.bfloat16, device=rt.device)       # padded columns are zero, as in the engine
    dzp[:, :n_out] = (torch.randn(rows, n_out, device=rt.device, generator=g) / rows).to(torch.bfloat16)
    wpad = torch.zeros(R, kt, device=rt.device)
    wpad[:n_out] = w
    img = torch.cat([C.pack_weight_f32(wpad[i * N:(i + 1) * N].contiguous(), N, False)[0] for i in range(n_imgs)])
    da = torch.full((rows, kt), float("nan"), dtype=torch.bfloat16, device=rt.device)
    C.sage_bwd_da(dzp, img, N, n_imgs, da)
    _within_ulp(da, dzp.float()[:, :n_out] @ w.to(torch.bfloat16).float())


def test_engine_uses_sage_bwd_da(rt):
    """Every layer l >= 2 of the supervised and link trainers takes dA_l from sage_bwd_da: L persistent-kernel launches
    (the forward), L - 1 sage_bwd_da launches, 9 / 12 / 14 launches per step for the 2-layer supervised and link trainers
    and a 3-layer trainer with an N-split 172-class top layer."""
    from torch.profiler import ProfilerActivity, profile

    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    torch.manual_seed(0)
    sup = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2).to(rt.device), [25, 10], 256, use_cuda_graph=False)
    link = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 64, 2).to(rt.device), [25, 10], 128, 5,
                               use_cuda_graph=False)
    deep = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 172, 3).to(rt.device), [5, 4, 3], 128,
                           use_cuda_graph=False)
    assert deep.n_split[-1] > 1
    e = (torch.randint(0, 20000, (128,)), torch.randint(0, 20000, (128,)))
    sup.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    deep.seeds.copy_(torch.randint(0, 20000, (128,), device=rt.device))
    for tr, step, n_launch in ((sup, sup._step_body, 9), (link, lambda: link.step(*e), 12), (deep, deep._step_body, 14)):
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if ev.device_type is not None and str(ev.device_type).endswith("CUDA")
                 and "glb::" in ev.name]
        assert len(names) == n_launch, names
        assert sum("sage_bwd_da_kernel" in n for n in names) == tr.L - 1, names
        assert sum("sage_persist_kernel" in n for n in names) == tr.L, names
        for da in tr.dA[1:]:
            assert torch.isfinite(da.float()).all() and da.abs().sum() > 0
