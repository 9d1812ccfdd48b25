"""Generate tests/golden/dense_weighted.pt by RUNNING THE REFERENCE'S OWN dense layer with softmax / softmin /
normalised_mean / identity.

    PYTHONPATH=. python tools/gen_golden_weighted.py          (needs the reference checkout, like oracle/gen_golden.py)

Reuses oracle/gen_golden.py's setup: the reference's files imported over the third-party shims of oracle/shims/
(PNA_REFERENCE overrides the checkout's location).  TEST INFRASTRUCTURE ONLY.
"""
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden import S3, DensePNALayer, dense_aggr, save  # noqa: E402

AGGRS = ["mean", "softmax", "softmin", "normalised_mean", "identity", "max"]
NEW = ("softmax", "softmin", "normalised_mean", "identity")


def one_case(adj, h, self_loop):
    """The reference's aggregators on X_j (reduce over dim 2), its layer's output, and its autograd gradients of h and of
    every parameter, in fp32 and in float64."""
    n = adj.size(1)
    f = h.size(2)
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    X_j = h.unsqueeze(1).repeat(1, n, 1, 1)
    k1 = {a: dense_aggr.AGGREGATORS[a](X_j, adj, self_loop=self_loop) for a in NEW}
    torch.manual_seed(7 + int(self_loop))
    lay = DensePNALayer(f, f, AGGRS, S3, avg_d, towers=2, self_loop=self_loop, pretrans_layers=1, posttrans_layers=1,
                        divide_input=True)
    lay.eval()
    with torch.no_grad():
        out = lay(h, adj)
    gw = torch.randn(out.shape, generator=torch.Generator().manual_seed(4))
    hg = h.clone().requires_grad_(True)
    lay.zero_grad()
    (lay(hg, adj) * gw).sum().backward()
    grads = dict(h=hg.grad.clone(), w=gw, params={k: v.grad.clone() for k, v in lay.named_parameters()})
    # the same layer in float64: what the fp32 results (the reference's and ours) are measured against
    lay64 = copy.deepcopy(lay).double()
    h64 = h.double().clone().requires_grad_(True)
    out64 = lay64(h64, adj.double())
    (out64 * gw.double()).sum().backward()
    grads64 = dict(h=h64.grad.clone(), params={k: v.grad.clone() for k, v in lay64.named_parameters()})
    return dict(avg_d=avg_d, k1=k1, out=out, grads=grads, out64=out64.detach(), grads64=grads64, state_dict=lay.state_dict(),
                ctor=dict(in_features=f, out_features=f, towers=2, self_loop=self_loop, pretrans_layers=1,
                          posttrans_layers=1, divide_input=True))


def weighted_case():
    """A directed 0/1 adjacency with a zero diagonal and at least one neighbour per row (so that the reference gives no
    NaN), moderate inputs, towers=2, once with self_loop=False and once with self_loop=True."""
    torch.manual_seed(41)
    B, n, f = 2, 16, 8
    adj = (torch.rand(B, n, n) < 0.25).float() * (1 - torch.eye(n))
    for b in range(B):
        for i in range(n):
            if adj[b, i].sum() == 0:
                adj[b, i, (i + 3) % n] = 1
    h = torch.randn(B, n, f)
    cases = {str(sl): one_case(adj, h, sl) for sl in (False, True)}
    save("dense_weighted", dict(kind="dense", adj=adj, h=h, aggregators=AGGRS, scalers=S3, cases=cases))


if __name__ == "__main__":
    weighted_case()
