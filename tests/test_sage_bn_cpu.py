"""EgoGraphSAGE(batch_norm=True) on the portable path: the layer structure, the bn -> ReLU order per hop tensor, the
running statistics of one BatchNorm1d call per hop tensor, eval mode and the momentum check."""
import pytest
import torch

from graphlearn_b200.models.graphsage import EgoGraphSAGE


def _xs(fan, B, d, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = [B]
    for k in fan:
        n.append(n[-1] * k)
    return [torch.randn(m, d, generator=g) * 3 + 5 for m in n]


def test_structure():
    m = EgoGraphSAGE(16, 32, 5, 3, batch_norm=True, bn_eps=1e-3, bn_momentum=0.2)
    assert len(m.norms) == 2
    assert all(n.num_features == 32 and n.eps == 1e-3 and n.momentum == 0.2 and n.affine and n.track_running_stats
               for n in m.norms)
    assert [c.bias is None for c in m.convs] == [True, True, False]
    plain = EgoGraphSAGE(16, 32, 5, 3)
    assert not hasattr(plain, "norms") and all(c.bias is not None for c in plain.convs)


@pytest.mark.parametrize("L,fan", [(2, [4, 3]), (3, [3, 2, 2])])
def test_dense_forward_is_bn_then_relu_per_hop_tensor(L, fan):
    torch.manual_seed(0)
    m = EgoGraphSAGE(8, 16, 4, L, batch_norm=True, bf16_activations=False)
    ref = [torch.nn.BatchNorm1d(16) for _ in range(L - 1)]
    for r, n in zip(ref, m.norms):
        r.load_state_dict(n.state_dict())
    xs = _xs(fan, 6, 8)
    out = m(xs, fan)
    h = xs
    for l in range(L):
        last = l == L - 1
        h = [m.convs[l](h[i], h[i + 1], fan[i]) for i in range(L - l)]
        if not last:
            h = [torch.relu(ref[l](z)) for z in h]
    torch.testing.assert_close(out, h[0])
    for l, n in enumerate(m.norms):
        assert int(n.num_batches_tracked) == L - l          # one update per hop tensor of the layer
        torch.testing.assert_close(n.running_mean, ref[l].running_mean)
        torch.testing.assert_close(n.running_var, ref[l].running_var)
    m.eval()
    before = [n.running_mean.clone() for n in m.norms]
    m(xs, fan)
    assert all(torch.equal(a, n.running_mean) for a, n in zip(before, m.norms))


@pytest.mark.parametrize("mom", [0.0, -0.1, 1.5])
def test_momentum_out_of_range_raises(mom):
    with pytest.raises(ValueError):
        EgoGraphSAGE(8, 16, 4, 2, batch_norm=True, bn_momentum=mom)
