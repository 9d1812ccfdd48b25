"""Generate tests/golden/dgl_edge_msgs.pt, dgl_edge_msgs_zinc.pt, dgl_edge_msgs_wide75.pt and pyg_edge_msgs.pt by RUNNING
THE REFERENCE'S OWN DGL PNALayer and PyG PNAConv with edge features and / or more than one pretrans layer -- the
configurations whose messages pna_edge_msg_fwd evaluates.

    PYTHONPATH=. python tools/gen_golden_edge_msgs.py          (needs the reference checkout, like oracle/gen_golden.py)

Reuses oracle/gen_golden.py's setup: the reference's files imported over the third-party shims of oracle/shims/
(PNA_REFERENCE overrides the checkout's location).  One random multigraph of 64 nodes with self loops, a duplicated edge,
in-degree-0 nodes and one row of in-degree 260 (above the split threshold, so the split-row merge runs).  Cases:
  DGL PNALayer  edge_features=True, pretrans_layers 1 / 2 / 3, divide_input both ways, towers 5 (in_dim 10, edge_dim 6);
                the README's ZINC shape (in_dim 70, edge_dim 50, towers 5, divide_input: F_t 14, L = 1);
                divide_input=False at in_dim 75 (F_t 75, above the 64 of the multi-layer kernel), L = 1, one tower,
                mean / max with the identity scaler (a small posttrans);
  PyG PNAConv   edge_dim 5 with pre_layers 1 / 2 / 3, divide_input both ways (12 -> 12, towers 2);
                pre_layers 3 without edge features.
As tools/gen_golden_pretrans.py, every bias is set to random values so that the ReLU boundaries are exercised.  Stores out
in fp32 and float64, the fp32 gradients of x / h and of edge_attr / e, and for every parameter its float64 gradient
(rounded to fp32) and the reference's own fp32 error against it.  The sizes are kept small so that each file stays a few
hundred KiB.  TEST INFRASTRUCTURE ONLY.
"""
import copy
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle.gen_golden import A4, S3, DGLPNALayer, PNAConv, deg_hist, dgl, graph_hub, save  # noqa: E402

N, E, HUB = 64, 100, 260


def _random_biases(lay):
    with torch.no_grad():
        for name, p in lay.named_parameters():
            if name.endswith("bias"):
                p.copy_(0.1 * torch.randn(p.shape))


def _run(lay, call, inputs, gw):
    """fp32 out (no grad) and float64 out; the fp32 gradients of the inputs; the float64 gradient of every parameter (stored
    rounded to fp32) and the reference's own fp32 error against it (relative Frobenius norm, computed in float64)."""
    with torch.no_grad():
        out = call(lay, *inputs)
    ins = [None if t is None else t.clone().requires_grad_(True) for t in inputs]
    lay.zero_grad()
    (call(lay, *ins) * gw).sum().backward()
    lay64 = copy.deepcopy(lay).double()
    ins64 = [None if t is None else t.double().clone().requires_grad_(True) for t in inputs]
    out64 = call(lay64, *ins64)
    (out64 * gw.double()).sum().backward()
    g32, g64 = dict(lay.named_parameters()), dict(lay64.named_parameters())
    ref_err = {k: float((g32[k].grad.double() - g64[k].grad).norm() / g64[k].grad.norm().clamp(min=1e-6)) for k in g64}
    return dict(out=out, out64=out64.detach().clone(), input_grads=[None if t is None else t.grad.clone() for t in ins],
                params64={k: v.grad.float().clone() for k, v in g64.items()}, ref_err=ref_err, w=gw,
                state_dict={k: v.clone() for k, v in lay.state_dict().items()})


def _inputs(ei, width, edge_dim, seed):
    """Node features, edge features (None without) and the output weights of one fixture file: every case of a file shares
    them, so torch.save stores them once."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, width, generator=g)
    e = torch.randn(ei.size(1), edge_dim, generator=g) if edge_dim else None
    return x, e, torch.randn(N, width, generator=g)


def dgl_case(ei, inputs, towers, divide_input, pretrans_layers, seed, aggr="mean max min std",
             scal="identity amplification attenuation"):
    torch.manual_seed(seed)
    h, e, gw = inputs
    in_dim, edge_dim = h.size(1), e.size(1)
    indeg = torch.bincount(ei[1], minlength=N).float()
    avg_d = dict(lin=indeg.mean().item(), exp=1.0, log=torch.log(indeg + 1).mean().item())
    snorm = torch.full((N, 1), 1.0 / np.sqrt(N))
    ctor = dict(in_dim=in_dim, out_dim=in_dim, dropout=0.0, graph_norm=True, batch_norm=True, residual=True, towers=towers,
                divide_input=divide_input, edge_features=True, edge_dim=edge_dim, pretrans_layers=pretrans_layers,
                posttrans_layers=1)
    lay = DGLPNALayer(aggregators=aggr, scalers=scal, avg_d=avg_d, **ctor)
    _random_biases(lay)
    lay.eval()
    call = lambda m, h_, e_: m(dgl.DGLGraph(ei[0], ei[1], N), h_, e_, snorm.to(h_.dtype))
    r = _run(lay, call, [h, e], gw)
    r.update(h=h, e=e, snorm_n=snorm, avg_d=avg_d, aggregators=aggr, scalers=scal, ctor=ctor)
    return r


def pyg_case(ei, inputs, towers, divide_input, pre_layers, seed):
    torch.manual_seed(seed)
    x, ea, gw = inputs
    fin, edge_dim = x.size(1), None if ea is None else ea.size(1)
    deg = deg_hist(ei[1], N)
    ctor = dict(in_channels=fin, out_channels=fin, edge_dim=edge_dim, towers=towers, pre_layers=pre_layers, post_layers=1,
                divide_input=divide_input)
    conv = PNAConv(aggregators=A4, scalers=S3, deg=deg, **ctor)
    _random_biases(conv)
    call = lambda m, x_, ea_: m(x_, ei, ea_)
    r = _run(conv, call, [x, ea], gw)
    r.update(x=x, edge_attr=ea, deg=deg, aggregators=A4, scalers=S3, ctor=ctor)
    return r


def main():
    ei = graph_hub(N, E, HUB, seed=21)
    indeg = torch.bincount(ei[1], minlength=N)
    assert int(indeg.min()) == 0 and int(indeg.max()) >= 256
    cases, seed, inputs = {}, 300, _inputs(ei, 10, 6, 1)
    for L in (1, 2, 3):
        for div in (True, False):
            cases[f"L{L}_div{int(div)}"] = dgl_case(ei, inputs, 5, div, L, seed)
            seed += 10
    save("dgl_edge_msgs", dict(kind="dgl_layer", edge_index=ei, cases=cases))
    save("dgl_edge_msgs_zinc", dict(kind="dgl_layer", edge_index=ei, cases={
        "zinc": dgl_case(ei, _inputs(ei, 70, 50, 2), 5, True, 1, seed)}))
    save("dgl_edge_msgs_wide75", dict(kind="dgl_layer", edge_index=ei, cases={
        "wide75": dgl_case(ei, _inputs(ei, 75, 4, 3), 1, False, 1, seed + 10, "mean max", "identity")}))
    cases, seed, inputs = {}, 500, _inputs(ei, 12, 5, 4)
    for L in (1, 2, 3):
        for div in (True, False):
            cases[f"edge_L{L}_div{int(div)}"] = pyg_case(ei, inputs, 2, div, L, seed)
            seed += 10
    cases["noedge_L3"] = pyg_case(ei, (inputs[0], None, inputs[2]), 2, False, 3, seed)
    save("pyg_edge_msgs", dict(kind="pyg_conv", edge_index=ei, cases=cases))


if __name__ == "__main__":
    main()
