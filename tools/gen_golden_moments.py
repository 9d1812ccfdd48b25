"""Generate tests/golden/dense_moments.pt by RUNNING THE REFERENCE'S OWN dense layer with the moment aggregators.

    PYTHONPATH=. python tools/gen_golden_moments.py          (needs the reference checkout, like oracle/gen_golden.py)

Reuses oracle/gen_golden.py's setup: the reference's files imported over the third-party shims of oracle/shims/
(PNA_REFERENCE overrides the checkout's location).  TEST INFRASTRUCTURE ONLY.
"""
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden import S3, DensePNALayer, dense_aggr, save  # noqa: E402


def moments_case():
    """The dense layer with the three central moments (models/pytorch/pna/aggregators.py:122-146) among six aggregators,
    towers=2, self_loop=False, on a directed 0/1 adjacency with at least 3 neighbours per row; plus the reference's moment aggregators on
    X_j (reduce over dim 2) and the reference-autograd gradients of h and every parameter."""
    torch.manual_seed(31)
    B, n, f = 2, 16, 8
    adj = (torch.rand(B, n, n) < 0.3).float() * (1 - torch.eye(n))
    for b in range(B):
        for i in range(n):
            # at least 3 neighbours per row: an odd central moment of 2 values is exactly 0, where sign(M_k) -- and so r_k,
            # by +-(1e-5)^(1/k) -- is decided by rounding in any fp32 evaluation, the reference's included
            for step in (1, 2, 3):
                if adj[b, i].sum() < 3:
                    adj[b, i, (i + step) % n] = 1
            if adj[b, :, i].sum() == 0:
                adj[b, (i + 2) % n, i] = 1
    h = torch.randn(B, n, f)
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    aggrs = ["mean", "max", "moment3", "moment4", "moment5", "std"]
    X_j = h.unsqueeze(1).repeat(1, n, 1, 1)
    k1 = {f"moment{k}": dense_aggr.AGGREGATORS[f"moment{k}"](X_j, adj) for k in (3, 4, 5)}
    lay = DensePNALayer(f, f, aggrs, S3, avg_d, towers=2, self_loop=False, pretrans_layers=1, posttrans_layers=1,
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
    save("dense_moments", dict(kind="dense", adj=adj, h=h, avg_d=avg_d, aggregators=aggrs, scalers=S3, k1=k1, grads=grads,
                               out64=out64.detach(), grads64=grads64,
                               ctor=dict(in_features=f, out_features=f, towers=2, self_loop=False, pretrans_layers=1,
                                         posttrans_layers=1, divide_input=True), state_dict=lay.state_dict(), out=out))


if __name__ == "__main__":
    moments_case()
