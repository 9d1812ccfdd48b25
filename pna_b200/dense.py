"""Dense-adjacency signature ``forward(input[B,N,F], adj[B,N,N])`` of the multitask loop
(reference ``models/pytorch/pna/layer.py``, called through ``models/pytorch/gnn_framework.py:94``) on the CSR kernel.

The reference builds a B x N x N x 2F pair tensor per layer application (layer.py:37-40) and reduces it with masked
dense sums (aggregators.py:17-84): O(B N^2 F).  Here ``adj`` becomes a block-diagonal edge list once per batch
(``adj[b,i,j] != 0`` => edge j -> i, aggregators.py:24-27) and every layer application is two node-level GEMMs plus
kernel calls -- the same adjacency is reused by all N/2 repeated layers of the multitask model.

Faithful to a quirk of the reference: ``aggregate_max/min`` reduce over dim -3 (the FIRST node index,
aggregators.py:39,51) while ``mean/std/sum`` reduce over dim 2, so for node v
    mean/std see  pretrans([h_v, h_u])  over u with adj[v,u] != 0      (self first)
    max/min  see  pretrans([h_u, h_v])  over u with adj[u,v] >  0      (neighbour first)
Two kernel calls fill one output row (PNA_AGGR_SKIP keeps the other call's column slots).
``self_loop=True`` aggregates over adj + I while the scalers keep the loop-free row degree (``pna_agg_t.scaler_degree``);
``var`` is clamped at 0 as the reference does (PNA_FLAG_RELU_VAR).
A weighted adjacency (an entry other than 0 and 1, found in the same pass as the edges) is reproduced as the reference
computes it (aggregators.py:17-84, scalers.py:8-38): mean/sum/var/std weigh every message with a[i, j] and divide by
W_i = sum_j a[i, j]; max/min reduce over the entries a[u, v] > 0, unweighted; the scalers use the real D = adj.sum(-1)
(pna_aggregate_fwd_weighted: slot_weight / scaler_degree_f, DESIGN section 2 "Weighted adjacency").  It takes mean, std, sum, var, max, min and
identity (the other aggregators raise NotImplementedError), gives adj no gradient (an adj that requires grad raises), and a
non-finite entry raises ValueError.  Unlike the reference, which divides by zero, isolated nodes get PyG semantics (a
moment of a row without neighbours is 0; max/min without a positive entry are 0).
Every name of the reference registry (models/pytorch/pna/aggregators.py:149-152) is taken.
The moments reduce over dim 2 like mean/std (self first).  ``self_loop=True`` with a moment raises NotImplementedError:
the reference's ``aggregate_moment`` adds I to adj and then calls ``aggregate_mean(..., self_loop=True)``, which adds I
again, so its moments are centred on a mean that counts the self loop twice -- not a central moment of any edge set the
kernel can be given.
softmax / softmin / normalised_mean also reduce over dim 2 (self first) and take ``self_loop=True`` (the reference adds I
once).  Where they deliberately differ from the reference:
  * a row without neighbours gives 0 (the reference: 0/0 = NaN for softmax and softmin);
  * softmax / softmin are evaluated shifted by the row's max / min, so they stay finite where the reference's unshifted
    exp overflows (messages above ~88.7) or underflows to 0/0;
  * normalised_mean weighs with D_k^(-1/2) of the aggregated row degrees (adj + I with ``self_loop``); a graph with an
    isolated node makes the reference's every row NaN (inf * 0 in its diagonal matmul), here that node just has weight 0.
``identity`` is X_ii = pretrans([h_i, h_i]) whatever adj says: no kernel call, its column slots are filled here (both
paths, autograd for its gradient) with the kernels' scaler factors of the loop-free row degree.

``pretrans_layers = L >= 2`` (a ReLU between the layers, so the message is no longer affine): the first layer still
splits into the node GEMMs A, Bm, b1 (packed as for the tower layers, towers.py), and ``pna_edge_mlp_fwd``
(edge_mlp.py) evaluates the rest of the chain once per edge of the row CSR, writing M [E, T*F_t] in slot order.  The
self-first aggregators read M in CSR order (normalised_mean with ``degree_col = row.col``); max/min read the same
messages through a third CSR (destination j, sources = the row-slot ids of the edges (i, j)), because X[u, v] of the
colwise reduction is the message of edge (u, v); ``identity`` runs the pretrans MLP on [h_i, h_i] in torch.  Tower widths above 64 raise NotImplementedError.
Under ``torch.autocast("cuda")`` A and Bm reach the kernel at the boundary (DESIGN section 2): bf16 ones run
``pna_edge_msg_fwd_bf16`` (no edge term, pitch F_t: the arithmetic of ``pna_edge_mlp_fwd``), fp16 ones are upcast to fp32.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from .aggregate import aggregate_forward, at_boundary, pna_aggregate
from .csr import build_csr, tensor_version
from .edge_mlp import edge_mlp
from . import _lib, capture
from .nn_blocks import FCLayer, MLP
from .towers import first_layer_pack, hidden_pack

_SELF_FIRST = ("mean", "std", "sum", "var", "moment3", "moment4", "moment5", "softmax", "softmin", "normalised_mean")
_MOMENTS = ("moment3", "moment4", "moment5")
_NBR_FIRST = ("max", "min")
_ADJ_WEIGHT = ("mean", "std", "sum", "var", "max", "min", "identity")     # what a weighted adjacency takes


class DenseGraphs:
    """Block-diagonal CSRs of a dense batch: one for adj (row i gathers j) and one for adj^T.

    A weighted adjacency (an entry other than 0 and 1) also keeps ``row_weight``, the fp32 weight a[b, i, j] of every slot of
    ``row`` (a = adj, or adj + I with ``self_loop``), takes ``colwise`` over the entries a > 0 only (the reference's max/min
    mask), and gives the scalers the fp32 degree D = adj.sum(-1).  On a 0/1 adjacency ``row_weight`` is None and the CSRs and
    the int32 degree are what they always were."""

    def __init__(self, adj: torch.Tensor, self_loop: bool = False):
        capture.guard("DenseGraphs (the CSRs of a dense batch not seen before: adj.nonzero)")
        adj = adj.detach()          # graph constants, cached by data pointer: no autograd history (adj gets no gradient)
        B, N, _ = adj.shape
        a = adj
        if self_loop:
            a = adj + torch.eye(N, device=adj.device, dtype=adj.dtype).unsqueeze(0)
        # (a non-finite entry, an entry other than 0 and 1), copied to the host ahead of nonzero, whose synchronisation
        # also completes the copy: the check costs no synchronisation of its own
        flags = torch.stack([~torch.isfinite(adj).all(), ((adj != 0) & (adj != 1)).any()])
        host = torch.empty(2, dtype=torch.bool, pin_memory=adj.is_cuda)
        host.copy_(flags, non_blocking=True)
        b, i, j = (a != 0).nonzero(as_tuple=True)
        nonfinite, weighted = host.tolist()
        if nonfinite:
            raise ValueError("dense PNALayer: the adjacency has a non-finite entry")
        off = b * N
        self.B, self.N = B, N
        self.row = build_csr(j + off, i + off, B * N)        # destination i, sources j with adj[i, j] != 0
        self.row_weight = None
        self._pairs = None
        if not weighted:
            # the scalers always see D = adj.sum(-1) of the ORIGINAL adjacency (models/pytorch/pna/scalers.py:13,21,28,35):
            # no self loop, row degree -- also for the max/min blocks, which reduce over the other axis
            self.scaler_degree = (adj != 0).sum(-1).reshape(B * N).to(torch.int32).contiguous()
            self.colwise = build_csr(i + off, j + off, B * N)    # destination j, sources i with adj[i, j] != 0
            return
        self.scaler_degree = adj.float().sum(-1).reshape(B * N).contiguous()
        w = a[b, i, j].float()
        self.row_weight = w[self.row.perm.long()].contiguous()
        pos = w > 0
        self.colwise = build_csr(i[pos] + off[pos], j[pos] + off[pos], B * N)   # destination j, sources i with a[i, j] > 0

    @property
    def pairs(self):
        """Destination j, sources = the slot ids of ``row`` whose edge is (i, j) (n_src = E, ascending): the max/min CSR
        over per-edge messages in row-slot order (a weighted adjacency: the slots of positive weight).  Built on first use
        (pretrans_layers >= 2 only)."""
        if self._pairs is None:
            E, dev = self.row.n_edges, self.row.device
            slots, dst = torch.arange(E, device=dev), self.row.col.long()
            if self.row_weight is not None:
                keep = self.row_weight > 0
                slots, dst = slots[keep], dst[keep]
            self._pairs = build_csr(slots, dst, self.B * self.N, n_src=E)
            self._pairs.sources_unique = True       # every slot is the source of at most one pair
        return self._pairs


_CACHE = {}


def dense_graphs(adj: torch.Tensor, self_loop: bool) -> DenseGraphs:
    key = (adj.data_ptr(), tensor_version(adj), tuple(adj.shape), bool(self_loop), str(adj.device))
    hit = _CACHE.get(key)
    if hit is None:
        if len(_CACHE) > 8:
            _CACHE.clear()
        hit = (adj, DenseGraphs(adj, self_loop))
        _CACHE[key] = hit
    capture.pin(hit[1])
    return hit[1]


class PNATower(nn.Module):
    def __init__(self, in_features, out_features, aggregators, scalers, avg_d, self_loop, pretrans_layers, posttrans_layers,
                 device):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.pretrans = MLP(in_size=2 * in_features, hidden_size=in_features, out_size=in_features, layers=pretrans_layers,
                            mid_activation="relu", last_activation="none")
        self.posttrans = MLP(in_size=(len(aggregators) * len(scalers) + 1) * in_features, hidden_size=out_features,
                             out_size=out_features, layers=posttrans_layers, mid_activation="relu", last_activation="none")


class PNALayer(nn.Module):
    """reference models/pytorch/pna/layer.py:57-116; parameter names ``towers.{t}.{pretrans,posttrans}...``,
    ``mixing_network.linear``."""

    def __init__(self, in_features, out_features, aggregators, scalers, avg_d, towers=1, self_loop=False, pretrans_layers=1,
                 posttrans_layers=1, divide_input=True, device="cpu"):
        super().__init__()
        assert (not divide_input) or in_features % towers == 0
        assert out_features % towers == 0
        self.aggregators, self.scalers = list(aggregators), list(scalers)
        for a in self.aggregators:
            if a not in _SELF_FIRST + _NBR_FIRST + ("identity",):
                raise KeyError(f"aggregator {a!r} is not available on the CUDA path")
        if pretrans_layers > 1 and (in_features // towers if divide_input else in_features) > _lib.EDGE_MLP_MAX_WIDTH:
            raise NotImplementedError(f"dense PNALayer: pretrans_layers > 1 takes a tower input width of at most "
                                      f"{_lib.EDGE_MLP_MAX_WIDTH} (the edge-MLP kernel's limit)")
        if self_loop and any(a in _MOMENTS for a in self.aggregators):
            raise NotImplementedError("dense PNALayer: moment aggregators with self_loop=True are not supported (the reference "
                                      "centres them on a mean that counts the self loop twice; see the module docstring)")
        self.avg_d = {k: float(v) for k, v in avg_d.items()}
        self.self_loop = self_loop
        self.divide_input = divide_input
        self.input_tower = in_features // towers if divide_input else in_features
        self.output_tower = out_features // towers
        self.in_features, self.out_features = in_features, out_features
        self.towers = nn.ModuleList([
            PNATower(self.input_tower, self.output_tower, self.aggregators, self.scalers, avg_d, self_loop, pretrans_layers,
                     posttrans_layers, device) for _ in range(towers)])
        self.mixing_network = FCLayer(out_features, out_features, activation="LeakyReLU")

    def _halves(self, h):
        """A = h W_first^T, Bm = h W_second^T (+ bias folded where it is gathered), first/second = cat order."""
        it = self.input_tower
        Wa, Wb, b, _ = first_layer_pack([tw.pretrans.fully_connected[0].linear for tw in self.towers], it, 0, it,
                                        self.divide_input)
        return h @ Wa.t(), h @ Wb.t(), b

    def _columns(self, width, a2, device):
        """bool [width]: output columns of the list positions of ``a2`` that are not "_skip" (per tower: self block, then
        S x A blocks of F_t) -- those of the max/min call, or of ``identity``.  Made once per layer and device: a copy
        from host memory cannot run inside a CUDA graph capture."""
        key = (width, tuple(a2), str(device))
        masks = self.__dict__.setdefault("_column_masks", {})
        if key not in masks:
            capture.guard("dense PNALayer's column mask (a host-to-device copy)", "run one eager step of this layer first")
            T, Ft = len(self.towers), self.input_tower
            A, S = len(self.aggregators), len(self.scalers)
            m = torch.zeros(T, 1 + S * A, Ft, dtype=torch.bool)
            for s_ in range(S):
                for a_, name in enumerate(a2):
                    if name != "_skip":
                        m[:, 1 + s_ * A + a_, :] = True
            masks[key] = m.reshape(-1)[:width].to(device)
        return masks[key]

    def forward(self, input, adj):
        B, N, Fin = input.shape
        graphs = dense_graphs(adj, self.self_loop)
        if graphs.row_weight is not None:
            bad = [a for a in self.aggregators if a not in _ADJ_WEIGHT]
            if bad:
                raise NotImplementedError(f"dense PNALayer: a weighted (non 0/1) adjacency takes the aggregators "
                                          f"{_ADJ_WEIGHT} only, not {bad}")
            if adj.requires_grad and torch.is_grad_enabled():
                raise ValueError("dense PNALayer: a weighted adjacency gets no gradient; pass adj.detach()")
        h = input.reshape(B * N, Fin)
        T = len(self.towers)
        a1 = [a if a in _SELF_FIRST else "_skip" for a in self.aggregators]
        a2 = [a if a in _NBR_FIRST else "_skip" for a in self.aggregators]
        nbr = any(a != "_skip" for a in a2)
        common = dict(towers=T, self_feat=h, self_divided=self.divide_input, relu_var=True,
                      scaler_degree=graphs.scaler_degree)
        rw = dict(slot_weight=graphs.row_weight) if graphs.row_weight is not None else {}
        if not self.towers[0].pretrans.is_single_affine():
            out, out2, x_id = self._forward_edge_mlp(h, graphs, a1, a2, nbr, common, rw)
        else:
            A, Bm, b = self._halves(h)
            out2, x_id = None, lambda: A + Bm + b
            if not (torch.is_grad_enabled() and (h.requires_grad or any(p.requires_grad for p in self.parameters()))):
                # mean/std: message = W_first h_v + W_second h_u + b, neighbours u from row v of adj
                out = aggregate_forward(Bm + b, graphs.row, a1, self.scalers, self.avg_d, row_bias=A, **common, **rw)
                # max/min: message = W_first h_u + W_second h_v + b, neighbours u from column v of adj; fills the
                # skipped slots
                if nbr:
                    aggregate_forward(A + b, graphs.colwise, a2, self.scalers, self.avg_d, row_bias=Bm, out=out, **common)
            else:
                # training (multitask_benchmark/util/train.py:148): two differentiable calls, columns merged by a mask
                out = pna_aggregate(Bm + b, graphs.row, a1, self.scalers, self.avg_d, row_bias=A, **common, **rw)
                if nbr:
                    out2 = pna_aggregate(A + b, graphs.colwise, a2, self.scalers, self.avg_d, row_bias=Bm, **common)
        if out2 is not None:
            both = any(a != "_skip" for a in a1)
            out = torch.where(self._columns(out.size(1), a2, h.device), out2, out) if both else out2
        if "identity" in self.aggregators:
            # X_ii = pretrans([h_i, h_i]) per tower, in every scaler's slot; autograd carries its gradient
            ident = [a if a == "identity" else "_skip" for a in self.aggregators]
            out = torch.where(self._columns(out.size(1), ident, h.device), self._identity_block(x_id(), graphs), out)
        # both calls scale with the ROW degree D = adj.sum(-1) of the loop-free adjacency (scaler_degree), as
        # models/pytorch/pna/scalers.py:13,21 does, whatever edge set the aggregators reduced over
        out = out.view(B * N, T, -1)
        y = torch.cat([tw.posttrans(out[:, t]) for t, tw in enumerate(self.towers)], dim=1)
        return self.mixing_network(y).view(B, N, -1)

    def _forward_edge_mlp(self, h, graphs, a1, a2, nbr, common, rw):
        """pretrans_layers >= 2: per-edge messages from pna_edge_mlp_fwd (module docstring) and their aggregation.  Returns
        the self-first aggregate, the neighbour-first one (None without max/min) and a callable giving the identity
        block's pretrans([h_i, h_i]); ``forward`` merges them as on the affine path."""
        if not all(tw.pretrans.is_linear_relu() for tw in self.towers):
            raise NotImplementedError("dense PNALayer: the edge-MLP kernel takes Linear/ReLU pretrans layers only")
        A, Bm, b1 = self._halves(h)
        W, bW = hidden_pack([[fc.linear for fc in tw.pretrans.fully_connected] for tw in self.towers])
        M = edge_mlp(at_boundary(A), at_boundary(Bm), b1, W, bW, graphs.row, len(self.towers))
        # self first: row i reads the messages of its own slots; normalised_mean weighs slot s with D of col[s]
        dcol = graphs.row.col if "normalised_mean" in self.aggregators else None
        out = pna_aggregate(M, graphs.row, a1, self.scalers, self.avg_d, messages_in_csr_order=True, degree_col=dcol,
                            **common, **rw)
        # neighbour first: node v reduces X[u, v] = M[slot of edge (u, v)] over u
        out2 = pna_aggregate(M, graphs.pairs, a2, self.scalers, self.avg_d, **common) if nbr else None
        it = self.input_tower
        xs = [h[:, t * it:(t + 1) * it] if self.divide_input else h for t in range(len(self.towers))]
        return out, out2, lambda: torch.cat([tw.pretrans(torch.cat([x, x], 1)) for x, tw in zip(xs, self.towers)], 1)

    def _identity_block(self, x_id, graphs):
        """[B*N, T * (1 + S*A) * F_t]: x_id's tower slice times each scaler's factor in every (scaler, aggregator) slot; the
        factors are the aggregation epilogue's (common.cuh deg_scales: attenuation / inverse_linear are 1 where D == 0);
        D is the int32 row degree, or the fp32 adj.sum(-1) of a weighted adjacency."""
        T, Ft = len(self.towers), self.input_tower
        A, S = len(self.aggregators), len(self.scalers)
        D = graphs.scaler_degree.to(x_id.dtype)
        lg = torch.log(D + 1)
        one = torch.ones_like(D)
        avg_log, avg_lin = self.avg_d["log"], self.avg_d.get("lin", 1.0)
        # D != 0, not D > 0: a signed adjacency can have a row sum in (-1, 0), where the reference and the kernels' deg_scales_f
        # divide as usual
        fac = {"identity": one, "amplification": lg / avg_log, "attenuation": torch.where(D != 0, avg_log / lg, one),
               "linear": D / avg_lin, "inverse_linear": torch.where(D != 0, avg_lin / D, one)}
        f = torch.stack([fac[s_] for s_ in self.scalers], 1)                         # [B*N, S]
        v = x_id.view(-1, T, 1, 1, Ft) * f.view(-1, 1, S, 1, 1)                      # [B*N, T, S, 1, F_t]
        v = v.expand(-1, T, S, A, Ft).reshape(-1, T, S * A, Ft)
        return torch.cat([torch.zeros_like(v[:, :, :1]), v], 2).reshape(x_id.size(0), -1)

    def __repr__(self):
        return f"{self.__class__.__name__} ({self.in_features} -> {self.out_features})"
