"""Generate tests/golden/dense_pretrans.pt by RUNNING THE REFERENCE'S OWN dense layer with pretrans_layers 2 and 3.

    PYTHONPATH=. python tools/gen_golden_pretrans.py          (needs the reference checkout, like oracle/gen_golden.py)

Reuses oracle/gen_golden.py's setup: the reference's files imported over the third-party shims of oracle/shims/
(PNA_REFERENCE overrides the checkout's location).  One directed 0/1 adjacency with at least 3 neighbours per row, towers=2,
every combination of pretrans_layers (2, 3), divide_input (True, False), self_loop (False, True) and two groups of
aggregators (mean max min std sum var; moment3 softmax softmin normalised_mean identity max); the moment only
without self_loop (the dense layer refuses that pair).  Stores out and the gradients of h and of every parameter, in fp32
and float64.  TEST INFRASTRUCTURE ONLY.
"""
import copy
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden import S3, DensePNALayer, save  # noqa: E402

# two aggregator groups (a layer call packs at most PNA_MAX_AGGR = 6 names): eleven aggregators in all
GROUPS = {"plain": ["mean", "max", "min", "std", "sum", "var"],
          "addon": ["moment3", "softmax", "softmin", "normalised_mean", "identity", "max"]}


def one_case(adj, h, aggrs, pretrans_layers, divide_input, self_loop, seed):
    f = h.size(2)
    aggrs = [a for a in aggrs if not (self_loop and a.startswith("moment"))]
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    ctor = dict(in_features=f, out_features=f, towers=2, self_loop=self_loop, pretrans_layers=pretrans_layers,
                posttrans_layers=1, divide_input=divide_input)
    torch.manual_seed(seed)
    lay = DensePNALayer(aggregators=aggrs, scalers=S3, avg_d=avg_d, **ctor)
    # the reference's zero biases would leave the ReLU masks of the hidden layers untested at their boundary: random ones
    with torch.no_grad():
        for name, p in lay.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape))
    lay.eval()
    with torch.no_grad():
        out = lay(h, adj)
    gw = torch.randn(out.shape, generator=torch.Generator().manual_seed(seed + 1))
    hg = h.clone().requires_grad_(True)
    lay.zero_grad()
    (lay(hg, adj) * gw).sum().backward()
    grads = dict(h=hg.grad.clone(), w=gw, params={k: v.grad.clone() for k, v in lay.named_parameters()})
    lay64 = copy.deepcopy(lay).double()
    h64 = h.double().clone().requires_grad_(True)
    out64 = lay64(h64, adj.double())
    (out64 * gw.double()).sum().backward()
    grads64 = dict(h=h64.grad.clone(), params={k: v.grad.clone() for k, v in lay64.named_parameters()})
    return dict(aggregators=aggrs, avg_d=avg_d, ctor=ctor, out=out, grads=grads, out64=out64.detach(), grads64=grads64,
                state_dict=lay.state_dict())


def pretrans_case():
    torch.manual_seed(43)
    B, n, f = 2, 12, 8
    adj = (torch.rand(B, n, n) < 0.3).float() * (1 - torch.eye(n))
    for b in range(B):
        for i in range(n):
            k = 1
            while adj[b, i].sum() < 3:
                adj[b, i, (i + k) % n] = 1
                k += 2
            k = 1
            while adj[b, :, i].sum() < 3:      # max/min reduce over the first node index: no empty column either
                adj[b, (i + k) % n, i] = 1
                k += 2
    h = torch.randn(B, n, f)
    cases = {}
    seed = 100
    for L in (2, 3):
        for divide in (True, False):
            for loop in (False, True):
                for group, aggrs in GROUPS.items():
                    cases[f"L{L}_div{int(divide)}_loop{int(loop)}_{group}"] = one_case(adj, h, aggrs, L, divide, loop, seed)
                    seed += 10
    save("dense_pretrans", dict(kind="dense", adj=adj, h=h, scalers=S3, cases=cases))


if __name__ == "__main__":
    pretrans_case()
