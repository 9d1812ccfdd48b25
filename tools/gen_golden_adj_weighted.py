"""Generate tests/golden/dense_adj_weighted.pt by RUNNING THE REFERENCE'S OWN dense layer on a weighted adjacency (real
entries, a few negative): mean / max / min / std / sum / var with all five scalers.

    PYTHONPATH=. python tools/gen_golden_adj_weighted.py      (needs the reference checkout, like oracle/gen_golden.py)

Reuses oracle/gen_golden.py's setup: the reference's files imported over the third-party shims of oracle/shims/
(PNA_REFERENCE overrides the checkout's location).  TEST INFRASTRUCTURE ONLY.
"""
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden import DensePNALayer, save  # noqa: E402

AGGRS = ["mean", "max", "min", "std", "sum", "var"]
S5 = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]


def one_case(adj, h, self_loop, pretrans_layers, divide_input, aggregators=AGGRS):
    """The reference layer's output and its autograd gradients of h and of every parameter, in fp32 and in float64."""
    f = h.size(2)
    D = adj.sum(-1)
    avg_d = dict(lin=D.mean().item(), log=torch.log(D + 1).mean().item())
    torch.manual_seed(11 + 2 * int(self_loop) + 4 * pretrans_layers + int(divide_input))
    ctor = dict(in_features=f, out_features=f, towers=2, self_loop=self_loop, pretrans_layers=pretrans_layers,
                posttrans_layers=1, divide_input=divide_input)
    lay = DensePNALayer(aggregators=aggregators, scalers=S5, avg_d=avg_d, **ctor)
    lay.eval()
    with torch.no_grad():
        out = lay(h, adj)
    gw = torch.randn(out.shape, generator=torch.Generator().manual_seed(5))
    hg = h.clone().requires_grad_(True)
    lay.zero_grad()
    (lay(hg, adj) * gw).sum().backward()
    grads = dict(h=hg.grad.clone(), w=gw, params={k: v.grad.clone() for k, v in lay.named_parameters()})
    lay64 = copy.deepcopy(lay).double()
    h64 = h.double().clone().requires_grad_(True)
    out64 = lay64(h64, adj.double())
    (out64 * gw.double()).sum().backward()
    grads64 = dict(h=h64.grad.clone(), params={k: v.grad.clone() for k, v in lay64.named_parameters()})
    assert torch.isfinite(out).all() and torch.isfinite(out64).all()
    return dict(avg_d=avg_d, out=out, grads=grads, out64=out64.detach(), grads64=grads64, state_dict=lay.state_dict(),
                ctor=ctor, aggregators=aggregators, adj=adj)


def adjacency(B, n, g):
    """Directed, weights in [0.25, 2], ~10 % of the entries negative; every row keeps W_i >= 0.5 and D_i + 1 >= 1.5 and every
    row and column a positive entry, so that the reference is finite."""
    mask = (torch.rand(B, n, n, generator=g) < 0.3).float() * (1 - torch.eye(n))
    w = torch.rand(B, n, n, generator=g) * 1.75 + 0.25
    sign = torch.where(torch.rand(B, n, n, generator=g) < 0.1, -1.0, 1.0)
    adj = mask * w * sign
    for b in range(B):
        for i in range(n):
            adj[b, i, (i + 5) % n] = 1.0 + 0.5 * (i % 3)          # a positive entry in every row and every column
            while adj[b, i].sum() < 0.5 or adj[b, i].sum() + 1 < 1.5:
                j = int(torch.randint(0, n, (1,), generator=g))
                if j != i and adj[b, i, j] < 0:
                    adj[b, i, j] = -adj[b, i, j]
    assert (adj > 0).any(2).all() and (adj > 0).any(1).all() and (adj < 0).any()
    return adj


def main():
    g = torch.Generator().manual_seed(43)
    B, n, f = 2, 16, 8
    adj = adjacency(B, n, g)
    h = torch.randn(B, n, f, generator=g)
    cases = {}
    for sl in (False, True):
        for L in (1, 2):
            for div in (True, False):
                cases[f"{sl}_{L}_{div}"] = one_case(adj, h, sl, L, div)
    # a row whose entries sum to D in (-1, 0): the scalers divide by log(D + 1) < 0 and by D < 0 (attenuation and
    # inverse_linear are 1 only where D == 0), also in the identity block; it keeps a positive entry for max / min
    neg = adj.clone()
    neg[0, 3] = 0
    neg[0, 3, 8], neg[0, 3, 10] = 0.5, -0.9
    assert -1 < float(neg[0, 3].sum()) < 0
    for L in (1, 2):
        cases[f"negD_{L}"] = one_case(neg, h, False, L, True, aggregators=["identity", "mean", "max", "std"])
    save("dense_adj_weighted", dict(kind="dense", adj=adj, h=h, aggregators=AGGRS, scalers=S5, cases=cases))


if __name__ == "__main__":
    main()
