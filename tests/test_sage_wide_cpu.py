"""Which GraphSAGE layer shapes the fused trainers run in one launch, split-K (two launches of kp = K / 2), or refuse
(ops.sage.fused_layer_plan); fused_supported keeps its one-launch meaning."""
import pytest
import torch

from graphlearn_b200.ops import sage as S


@pytest.mark.parametrize("agg", ["mean", "sum", "max"])
@pytest.mark.parametrize("d", [257, 264, 300, 384, 500, 512])
def test_wide_inputs_split(agg, d):
    """inputs 257-512 wide pad each half to 512: K = 1024 never fits one launch, each half of 512 does"""
    assert not S.fused_supported(d, d, 47, agg, 10)
    assert S.fused_layer_plan(d, d, 47, agg, 10, last=True) == (2, 1, 64)
    assert S.fused_layer_plan(d, d, 128, agg, 25) == (2, 2, 64)
    assert S.fused_layer_plan(d, d, 256, agg, 25) == (2, 4, 64)
    assert S.fused_layer_plan(d, d, 512, agg, 63) == (2, 8, 64)
    assert S.fused_layer_plan(d, d, 172, agg, 10, last=True) == (2, 3, 64)


@pytest.mark.parametrize("d,out,agg,k,last,plan", [
    (100, 47, "mean", 25, True, (1, 1, 64)),          # the headline shape: one launch, unchanged
    (100, 256, "max", 25, False, (1, 1, 256)),
    (100, 512, "mean", 10, False, (1, 2, 256)),       # a 512-wide hidden output over a 100-wide input: one launch
    (256, 256, "sum", 10, False, (1, 4, 64)),
    (256, 172, "max", 5, True, (1, 3, 64)),
    (300, 47, "gcn", 25, True, (1, 1, 64)),           # gcn has one half: K = 512 still fits
    (512, 256, "gcn", 10, False, (1, 4, 64)),
])
def test_one_launch_shapes(d, out, agg, k, last, plan):
    assert S.fused_layer_plan(d, d, out, agg, k, last=last) == plan
    assert S.fused_supported(d, d, min(out, plan[2]), agg, k)


def test_one_launch_plan_is_the_old_check():
    """wherever the old check (weight fits one launch, a hidden N-split is even, fused_supported) accepts a layer, the
    plan is one launch with the same images; wherever it refuses, the plan is split-K or a ValueError"""
    for d in (1, 8, 64, 100, 128, 200, 256, 257, 300, 512):
        for out in (1, 40, 47, 64, 128, 172, 256, 300, 512):
            for agg in ("mean", "sum", "max", "gcn"):
                for k in (1, 10, 15, 25, 31, 63, 64):
                    for last in (False, True):
                        kt = sum(S.padded_dims(d, d, agg))
                        ns, N = S.split_images(kt, out)
                        old = S.smem_fits(kt, N) and (ns == 1 or last or ns * N == out) and \
                            S.fused_supported(d, d, min(out, N), agg, k)
                        try:
                            plan = S.fused_layer_plan(d, d, out, agg, k, last=last)
                        except ValueError:
                            plan = None
                        if old:
                            assert plan == (1, ns, N), (d, out, agg, k, last, plan)
                        else:
                            assert plan is None or plan[0] == 2, (d, out, agg, k, last, plan)
                        if plan is not None and plan[0] == 2:
                            assert d > 256 and agg != "gcn", (d, out, agg, k, last, plan)


def test_fused_supported_values_unchanged():
    assert S.fused_supported(100, 100, 47, "mean", 25)
    assert S.fused_supported(256, 256, 64, "max", 25)
    assert S.fused_supported(512, 512, 64, "gcn", 63)
    assert not S.fused_supported(512, 512, 64, "gcn", 64)
    assert not S.fused_supported(600, 600, 47, "mean", 10)
    assert not S.fused_supported(300, 300, 47, "mean", 10)
    assert not S.fused_supported(64, 64, 47, "mean", 16)      # 4 rows per item: k + 1 <= 16
    assert S.fused_supported(64, 64, 47, "mean", 15)
    assert S.fused_supported(64, 64, 47, "mean", 31, torch.float32)
    assert S.split_images(1024, 256) == (8, 32) and not S.smem_fits(1024, 32)
    assert S.split_images(512, 256) == (4, 64) and S.smem_fits(512, 64)
    assert [S.max_fanout(kp) for kp in (64, 128, 256, 512)] == [15, 31, 63, 63]
    assert [S.max_fanout(kp, torch.float32) for kp in (64, 128, 256, 512)] == [31, 63, 63, 63]


def test_rejections_name_the_limit():
    with pytest.raises(ValueError, match="fan-out 64 exceeds the limit of 63"):
        S.fused_layer_plan(300, 300, 256, "mean", 64)
    with pytest.raises(ValueError, match="hidden width 300 does not split evenly over 5 weight images of 64 columns"):
        S.fused_layer_plan(300, 300, 300, "max", 10)
    with pytest.raises(ValueError, match="does not split evenly"):
        S.fused_layer_plan(100, 100, 300, "mean", 10)
    with pytest.raises(ValueError, match="inputs up to 512 wide"):
        S.fused_layer_plan(600, 600, 47, "mean", 10)
    with pytest.raises(ValueError, match="unknown aggregation"):
        S.fused_layer_plan(100, 100, 47, "lstm", 10)
    assert S.fused_layer_plan(300, 300, 300, "max", 10, last=True) == (2, 5, 64)     # a top layer may be split unevenly
