"""DGL-signature PNA layers (reference ``models/dgl/pna_layer.py``) on the sm_90a aggregation kernel.

Same constructors, same ``forward(g, h, e, snorm_n)`` / ``forward(g, h)``, same parameter names
(``towers.{t}.pretrans.fully_connected.{k}.linear``, ``...posttrans...``, ``towers.{t}.batchnorm_h``,
``mixing_network.linear``; ``posttrans`` / ``batchnorm_h`` for the simple layer).  ``g`` is duck-typed (graph.py).
DGL's ``apply_edges`` + ``update_all`` with a Python reduce UDF per in-degree bucket (pna_layer.py:61-64,202) is
replaced by ONE kernel call over all towers; in-degree-0 nodes keep DGL's zero rows (PNA_FLAG_ZERO_ISOLATED).

``PNALayer`` messages (pna_layer.py:35-40, ``pretrans(cat[src h, dst h, ef])``): without edge features and with one
pretrans layer they are affine and never built (two node GEMMs and the aggregation's row bias).  With edge features or
``pretrans_layers > 1`` they are written once, in CSR slot order at the padded tower width, by ``pna_edge_msg_fwd``
(edge_mlp.py): node GEMMs for the source and destination halves of the first pretrans Linear, one GEMM of the permuted
``ef`` against every tower's edge columns, and the rest of the pretrans MLP per edge.  The towers' ``pretrans`` run in
torch on gathered rows only for inputs the kernel does not take: dtypes other than float32, ``pretrans_layers > 1`` with
a tower width above 64, pretrans stacks that are not plain Linear / ReLU (dropout or batch norm inside), and training
steps on graphs below ``edge_mlp.FUSED_TRAINING_MIN_EDGES`` edges, where the torch path measured faster.  This message and
aggregation path, and the weight packs it caches, are shared with ``PNAConv`` (towers.py).

Under ``torch.autocast("cuda")`` ``PNALayer`` hands its GEMM products to the kernels in ``aggregate.boundary_dtype()``
(DESIGN section 2): bf16 operands run the bf16 aggregation, messages and compact tower post-linear whatever h's dtype, fp16
ones are upcast to fp32.  The tower width is padded for that dtype; the weights stay fp32.
"""
from __future__ import annotations

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import padding as pad
from .aggregate import pna_aggregate, row_scales
from .edge_mlp import edge_messages
from .linear import compact_path_ok, post_linear_towers_scaled
from .graph import graph_csr
from .static_batch import StaticBatch
from .nn_blocks import FCLayer, MLP
from .towers import TowerLayer

_AGGRS = ("mean", "sum", "max", "min", "std", "var")       # models/dgl/aggregators.py:50-52 minus moment3/4/5
_SCALERS = ("identity", "amplification", "attenuation")     # models/dgl/scalers.py:22


def _split(names, allowed, what):
    names = names.split() if isinstance(names, str) else list(names)
    for n in names:
        if n not in allowed:
            raise KeyError(f"{what} {n!r} is not available on the CUDA path (supported: {allowed})")
    return names


def _avg(avg_d) -> dict:
    return {k: float(v) for k, v in avg_d.items()}


class PNATower(nn.Module):
    """Parameters of one tower (pna_layer.py:17-33).  The aggregation itself runs once for all towers in PNALayer."""

    def __init__(self, in_dim, out_dim, dropout, graph_norm, batch_norm, aggregators, scalers, avg_d, pretrans_layers,
                 posttrans_layers, edge_features, edge_dim):
        super().__init__()
        self.dropout, self.graph_norm, self.batch_norm, self.edge_features = dropout, graph_norm, batch_norm, edge_features
        self.in_dim = in_dim
        self.batchnorm_h = nn.BatchNorm1d(out_dim)
        self.pretrans = MLP(in_size=2 * in_dim + (edge_dim if edge_features else 0), hidden_size=in_dim, out_size=in_dim,
                            layers=pretrans_layers, mid_activation="relu", last_activation="none")
        self.posttrans = MLP(in_size=(len(aggregators) * len(scalers) + 1) * in_dim, hidden_size=out_dim, out_size=out_dim,
                             layers=posttrans_layers, mid_activation="relu", last_activation="none")

    def finish(self, h_cat, snorm_n, blocks=None, fp=None, g=None):
        """posttrans -> graph norm -> batch norm -> dropout (pna_layer.py:67-76).  h_cat may carry padded column blocks
        (width fp instead of in_dim): the first posttrans Linear then gets zero weight columns at the pad positions."""
        if fp is not None and fp != self.in_dim:
            w0 = pad.expand_weight_cols(self.posttrans.fully_connected[0].linear.weight, blocks, self.in_dim, fp)
            h = self.posttrans(h_cat, first_weight=w0)
        else:
            h = self.posttrans(h_cat)
        return self._norms(h, snorm_n, g)

    def finish_linear(self, h, snorm_n, g=None):
        """``finish`` from the output of the first posttrans Linear (computed for every tower at once by PNALayer)."""
        fcs = self.posttrans.fully_connected
        h = fcs[0].after_linear(h)
        for fc in list(fcs)[1:]:
            h = fc(h)
        return self._norms(h, snorm_n, g)

    def _norms(self, h, snorm_n, g=None):
        if self.graph_norm:
            h = h * snorm_n
        if self.batch_norm:     # a StaticBatch: statistics over its real rows only
            h = g.batch_norm(self.batchnorm_h, h) if isinstance(g, StaticBatch) else self.batchnorm_h(h)
        return F.dropout(h, self.dropout, training=self.training)


class PNALayer(TowerLayer, nn.Module):
    """reference pna_layer.py:79-148."""

    def __init__(self, in_dim, out_dim, aggregators, scalers, avg_d, dropout, graph_norm, batch_norm, towers=1,
                 pretrans_layers=1, posttrans_layers=1, divide_input=True, residual=False, edge_features=False, edge_dim=0):
        super().__init__()
        assert (not divide_input) or in_dim % towers == 0, "if divide_input is set the number of towers has to divide in_dim"
        assert out_dim % towers == 0, "the number of towers has to divide the out_dim"
        assert avg_d is not None
        self.aggregators = _split(aggregators, _AGGRS, "aggregator")
        self.scalers = _split(scalers, _SCALERS, "scaler")
        self.avg_d = _avg(avg_d)
        self.divide_input = divide_input
        self.input_tower = in_dim // towers if divide_input else in_dim
        self.output_tower = out_dim // towers
        self.in_dim, self.out_dim = in_dim, out_dim
        self.edge_features = edge_features
        self.residual = residual and in_dim == out_dim
        self.towers = nn.ModuleList([
            PNATower(in_dim=self.input_tower, out_dim=self.output_tower, aggregators=self.aggregators, scalers=self.scalers,
                     avg_d=avg_d, pretrans_layers=pretrans_layers, posttrans_layers=posttrans_layers, batch_norm=batch_norm,
                     dropout=dropout, graph_norm=graph_norm, edge_features=edge_features, edge_dim=edge_dim)
            for _ in range(towers)])
        self.mixing_network = FCLayer(out_dim, out_dim, activation="LeakyReLU")

    n_towers = property(lambda self: len(self.towers))
    tower_in = property(lambda self: self.input_tower)
    avg = property(lambda self: self.avg_d)

    # -- what differs from PNAConv on the shared tower path (towers.py) -------------------------------------------------
    _SRC_FIRST = True                                   # pretrans(cat[src h, dst h, ef]) (pna_layer.py:35-40)
    _AGG_FLAGS = dict(zero_isolated=True, relu_var=True)

    def _pre_linears(self):
        return [[fc.linear for fc in tw.pretrans.fully_connected] for tw in self.towers]

    def _post_linears(self):
        return [tw.posttrans.fully_connected[0].linear for tw in self.towers]

    def _affine(self, e) -> bool:
        return not self.edge_features and self.towers[0].pretrans.is_single_affine()

    def _fused_layer_ok(self, e, amp: bool) -> bool:
        """Linear/ReLU pretrans stacks (no dropout or batch norm inside), and ef when edge features are announced."""
        return ((not self.edge_features or (e is not None and (amp or e.dtype == torch.float32)))
                and all(tw.pretrans.is_linear_relu() for tw in self.towers))

    def _fused_messages(self, h, csr, e, fp: int):
        A, Bm, b1, W, bW, C = self._message_operands(h, csr, e if self.edge_features else None)
        return edge_messages(A, Bm, b1, W, bW, csr, len(self.towers), edge_term=C, pitch=fp)

    def _torch_messages(self, h, csr, e):
        return self._edge_messages(csr, h, e)

    def _tower_input(self, h, t):
        it = self.input_tower
        return h[:, t * it:(t + 1) * it] if self.divide_input else h

    def _edge_messages(self, csr, h, e):
        src, dst = csr.col.long(), csr.dst_of_slot
        ef = e.index_select(0, csr.perm.long()) if self.edge_features else None
        msgs = []
        for t, tw in enumerate(self.towers):
            ht = self._tower_input(h, t)
            parts = [ht.index_select(0, src), ht.index_select(0, dst)] + ([ef] if ef is not None else [])
            msgs.append(tw.pretrans(torch.cat(parts, dim=1)))
        return torch.cat(msgs, dim=1)

    def forward(self, g, h, e, snorm_n):
        h_in = h
        csr = graph_csr(g, h.device)
        fp = self._tower_pitch(h)
        agg, compact = self._aggregate_towers(h, csr, e, fp, self._self_features(h, fp))
        if compact:
            # the rest of each tower's posttrans and norms on its output_tower slice of the towers' first posttrans Linear
            y = post_linear_towers_scaled(agg, row_scales(csr, self.scalers, self.avg_d), *self._post_weights(fp))
            ot = self.output_tower
            h_cat = torch.cat([tw.finish_linear(y[:, t * ot:(t + 1) * ot], snorm_n, g) for t, tw in enumerate(self.towers)], dim=1)
        else:
            blocks = 1 + len(self.aggregators) * len(self.scalers)
            agg = agg.view(h.size(0), len(self.towers), -1)                # [N, T, (1 + S*A) * fp] = cat([h_t, reduced])
            h_cat = torch.cat([tw.finish(agg[:, t], snorm_n, blocks, fp, g) for t, tw in enumerate(self.towers)], dim=1)
        h_out = self.mixing_network(h_cat)
        if self.residual:
            h_out = h_in + h_out
        return h_out

    def __repr__(self):
        return f"{self.__class__.__name__}(in_channels={self.in_dim}, out_channels={self.out_dim})"


class PNASimpleLayer(nn.Module):
    """reference pna_layer.py:151-219: aggregate the neighbours' h directly, posttrans, BN, ReLU, residual, dropout."""

    def __init__(self, in_dim, out_dim, aggregators, scalers, avg_d, dropout, batch_norm, residual, posttrans_layers=1):
        super().__init__()
        self.aggregators = _split(aggregators, _AGGRS, "aggregator")
        self.scalers = _split(scalers, _SCALERS, "scaler")
        self.in_dim, self.out_dim = in_dim, out_dim
        self.dropout, self.batch_norm, self.residual = dropout, batch_norm, residual
        self.batchnorm_h = nn.BatchNorm1d(out_dim)
        self.posttrans = MLP(in_size=(len(self.aggregators) * len(self.scalers)) * in_dim, hidden_size=out_dim, out_size=out_dim,
                             layers=posttrans_layers, mid_activation="relu", last_activation="none")
        self.avg_d = _avg(avg_d)

    def aggregate_only(self, g, h):
        return pna_aggregate(h, graph_csr(g, h.device), self.aggregators, self.scalers, self.avg_d, zero_isolated=True, relu_var=True)

    def forward(self, g, h):
        h_in = h
        fp = pad.padded_width(self.in_dim, h.dtype)
        csr = graph_csr(g, h.device)
        blocks = len(self.aggregators) * len(self.scalers)
        w0 = self.posttrans.fully_connected[0].linear.weight
        if fp != self.in_dim:   # odd width: 128-bit path on zero-padded rows, padding absorbed by the first posttrans Linear
            w0 = pad.expand_weight_cols(w0, blocks, self.in_dim, fp)
        hp = pad.pad_cols(h, fp)
        if w0.dtype == torch.float32 and compact_path_ok(h, len(self.aggregators) * fp, w0.size(0), len(self.scalers)):
            # compact post path: identity-scaled aggregate, the scaled copies are formed inside the tensor-core linear
            agg = pna_aggregate(hp, csr, self.aggregators, ["identity"], self.avg_d, zero_isolated=True, relu_var=True)
            h = self.posttrans(agg, first_weight=w0, first_row_scale=row_scales(csr, self.scalers, self.avg_d))
        else:
            agg = pna_aggregate(hp, csr, self.aggregators, self.scalers, self.avg_d, zero_isolated=True, relu_var=True)
            h = self.posttrans(agg, first_weight=w0)
        if self.batch_norm:
            h = g.batch_norm(self.batchnorm_h, h) if isinstance(g, StaticBatch) else self.batchnorm_h(h)
        h = F.relu(h)
        if self.residual:
            h = h_in + h
        return F.dropout(h, self.dropout, training=self.training)

    def __repr__(self):
        return f"{self.__class__.__name__}(in_channels={self.in_dim}, out_channels={self.out_dim})"
