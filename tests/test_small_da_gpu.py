"""dA = dZ . W of a top layer of <= 64 output columns on the small mma.sync kernel (sage_bwd_da) over the layer's forward
weight image, against the persistent forward kernel over a W^T image (the general dA path) and an fp32 reference."""
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


@pytest.mark.parametrize("rows,n_out,kt", [(1024, 47, 512), (3584, 64, 512), (1000, 20, 256), (37, 64, 256)])
def test_sage_bwd_da_matches_general_path(rt, rows, n_out, kt):
    from graphlearn_b200.parallel.runtime import local_table_desc, native
    C = native()
    g = torch.Generator(device=rt.device).manual_seed(rows + n_out)
    w = torch.randn(n_out, kt, device=rt.device, generator=g) / math.sqrt(kt)
    dzp = torch.zeros(rows, 64, dtype=torch.bfloat16, device=rt.device)       # padded columns are zero, as in the engine
    dzp[:, :n_out] = (torch.randn(rows, n_out, device=rt.device, generator=g) / rows).to(torch.bfloat16)
    img, _ = C.pack_weight_f32(w.contiguous(), 64, False)
    da = torch.full((rows, kt), float("nan"), dtype=torch.bfloat16, device=rt.device)
    C.sage_bwd_da(dzp, img, 64, da)
    _within_ulp(da, dzp.float()[:, :n_out] @ w.to(torch.bfloat16).float())
    # the general path: persistent forward kernel over a K-major W^T image, one CTA image per 256 columns
    wt = C.pack_weight_t(w.contiguous(), 64, 256)
    ref = torch.zeros(rows, kt, dtype=torch.bfloat16, device=rt.device)
    d = local_table_desc(dzp)
    cols = min(256, kt)
    C.sage_fused_multi(d, d, [None], [None], [0], [0], [rows], [0], [ref[:, :cols]], [None], 0, wt, None, 256, cols,
                       False, True, [], 1, wt.size(0), 0)
    _within_ulp(da, ref.float())


def test_engine_top_layer_uses_small_da(rt):
    """The 2-layer supervised and link trainers take dA_L from sage_bwd_da (no W^T image for the top layer, no third
    persistent-kernel launch) and keep 9 / 12 launches per step."""
    from torch.profiler import ProfilerActivity, profile

    from graphlearn_b200.engine import FastLinkSageTrainer, FastSageTrainer
    from graphlearn_b200.models.graphsage import EgoGraphSAGE
    from graphlearn_b200.store.synthetic import make_sharded_graph
    nodes, csr = make_sharded_graph(rt, 20000, 300000, 100, 47, seed=0)
    torch.manual_seed(0)
    sup = FastSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 47, 2).to(rt.device), [25, 10], 256, use_cuda_graph=False)
    link = FastLinkSageTrainer(rt, nodes, csr, EgoGraphSAGE(100, 256, 64, 2).to(rt.device), [25, 10], 128, 5,
                               use_cuda_graph=False)
    e = (torch.randint(0, 20000, (128,)), torch.randint(0, 20000, (128,)))
    sup.seeds.copy_(torch.randint(0, 20000, (256,), device=rt.device))
    for tr, step, n_launch in ((sup, sup._step_body, 9), (link, lambda: link.step(*e), 12)):
        assert tr._small_top_da and tr.img_t[-1] is None
        step()
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            step()
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if ev.device_type is not None and str(ev.device_type).endswith("CUDA")
                 and "glb::" in ev.name]
        assert len(names) == n_launch, names
        assert sum("sage_bwd_da_kernel" in n for n in names) == 1 and sum("sage_persist_kernel" in n for n in names) == 2, names
        assert torch.isfinite(tr.dA[-1].float()).all() and tr.dA[-1].abs().sum() > 0
