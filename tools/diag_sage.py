"""Diagnostic for the wgmma fused SAGE kernel: structured inputs that expose
layout mistakes (swizzle, descriptor, accumulator fragment mapping) as recognisable patterns."""
import sys, os, math
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from graphlearn_b200.parallel.runtime import init
from graphlearn_b200.ops import sage as SG

rt = init()
dev = rt.device
torch.manual_seed(0)


def run(M, k, d, n_out, mode="mean", w=None, xs=None, xn=None, tag=""):
    xs = torch.randn(M, d, device=dev) if xs is None else xs
    xn = torch.randn(M * k, d, device=dev) if xn is None else xn
    kin = d if mode == "gcn" else 2 * d
    w = torch.randn(n_out, kin, device=dev) / math.sqrt(kin) if w is None else w
    y = SG.sage_layer(SG.pad_weight(w, d, d, mode), None, k=k, mode=mode, relu=False, x_self=xs, x_nbr=xn).float()
    torch.cuda.synchronize()
    ref = SG.sage_layer_reference(w, None, xs.to(torch.bfloat16).float(), xn, k, mode, False)
    err = (y - ref).abs()
    print("[%s] M=%d k=%d d=%d n_out=%d mode=%s  max_err=%.4g  ref_max=%.4g  bad=%d/%d" % (
        tag, M, k, d, n_out, mode, err.max().item(), ref.abs().max().item(), int((err > 0.05).sum()), err.numel()))
    if err.max() > 0.05:
        bad = (err > 0.05).nonzero()[:12]
        for r, c in bad.tolist():
            print("    y[%d,%d]=%.4f ref=%.4f" % (r, c, y[r, c].item(), ref[r, c].item()))
        badrows = (err > 0.05).any(1).nonzero().flatten()[:40].tolist()
        badcols = (err > 0.05).any(0).nonzero().flatten()[:40].tolist()
        print("    bad rows:", badrows)
        print("    bad cols:", badcols)
    return y, ref


# 1) identity weights: out[m, n] = x_self[m, n]  (n < 64) -> exposes A/B/accumulator mapping
d = 64
w = torch.zeros(64, 2 * d, device=dev)
w[torch.arange(64), torch.arange(64)] = 1.0
xs = (torch.arange(128, device=dev)[:, None] * 1.0 + torch.arange(d, device=dev)[None, :] / 128.0)
y, ref = run(128, 1, d, 64, w=w, xs=xs, tag="identity-self")
print("   y[0,:8]  =", y[0, :8].tolist())
print("   ref[0,:8]=", ref[0, :8].tolist())
print("   y[5,:8]  =", y[5, :8].tolist())
print("   ref[5,:8]=", ref[5, :8].tolist())
# 2) identity on the neighbour half
w2 = torch.zeros(64, 2 * d, device=dev)
w2[torch.arange(64), d + torch.arange(64)] = 1.0
run(128, 2, d, 64, w=w2, tag="identity-nbr")
# 3) random, growing shapes
run(128, 4, 64, 64, tag="rand-small")
run(128, 4, 100, 256, tag="rand-d100-n256")
run(300, 10, 100, 256, tag="rand-M300")
run(256, 25, 256, 47, tag="rand-d256-n47")
run(256, 5, 100, 64, mode="gcn", tag="gcn")
run(256, 5, 100, 128, mode="sum", tag="sum")
print("DIAG DONE")
