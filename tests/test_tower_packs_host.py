"""The weight packs of the shared tower path (pna_b200/towers.py) are the same for PNAConv and the DGL PNALayer when the
two hold the same weights: only the column order of the first pre Linear differs ([dst, src, e] against [src, dst, e])."""
import pytest
import torch

import pna_b200
from pna_b200 import padding as pad

AGGRS, SCALERS = ["mean", "max"], ["identity", "amplification"]


@pytest.mark.parametrize("divide", [True, False])
@pytest.mark.parametrize("towers", [1, 5])
@pytest.mark.parametrize("width", [16, 15])
def test_pyg_and_dgl_pack_the_same_weights_identically(divide, towers, width):
    torch.manual_seed(towers * 100 + width)
    F = width
    cin = towers * F if divide else F
    conv = pna_b200.PNAConv(cin, towers * 4, AGGRS, SCALERS, torch.tensor([0, 3, 5, 2]), edge_dim=3, towers=towers,
                            pre_layers=2, divide_input=divide)
    lay = pna_b200.PNALayer(cin, towers * 4, AGGRS, SCALERS, {"log": 1.5, "lin": 3.0}, 0.0, False, False, towers=towers,
                            pretrans_layers=2, divide_input=divide, edge_features=True, edge_dim=F)
    with torch.no_grad():
        for pre, post, tw in zip(conv.pre_nns, conv.post_nns, lay.towers):
            fcs = tw.pretrans.fully_connected
            w = pre[0].weight
            fcs[0].linear.weight.copy_(torch.cat([w[:, F:2 * F], w[:, :F], w[:, 2 * F:]], 1))     # [src, dst, e]
            fcs[0].linear.bias.copy_(pre[0].bias)
            fcs[1].linear.weight.copy_(pre[2].weight)
            fcs[1].linear.bias.copy_(pre[2].bias)
            tw.posttrans.fully_connected[0].linear.weight.copy_(post[0].weight)
            tw.posttrans.fully_connected[0].linear.bias.copy_(post[0].bias)
        fp = pad.padded_width(F, torch.float32)
        assert fp == 16
        for a, b in [(conv._uv_weights(fp), lay._uv_weights(fp)), (conv._message_weights(), lay._message_weights()),
                     (conv._post_weights(fp), lay._post_weights(fp))]:
            assert len(a) == len(b)
            for x, y in zip(a, b):
                assert torch.equal(x, y)
