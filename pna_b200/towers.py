"""The tower message path of ``PNAConv`` (pyg.py) and the DGL ``PNALayer`` (dgl_layers.py), and the pre Linear packing
the dense ``PNALayer`` (dense.py) uses too.

The two tower layers run one algorithm up to their first post Linear: self features at the padded tower width, the
compact post-path decision, the messages (affine U = x W_dst^T, V = x W_src^T + b out of one GEMM; else the fused
``edge_messages`` kernel or the layer's torch fallback) and one ``pna_aggregate`` over all towers.  ``TowerLayer`` holds
it; each layer keeps its Linear accessors, column order, edge rows, torch fallback, and all that follows the first post
Linear.  Every weight pack is cached by ``cached``.
"""
from __future__ import annotations

import torch

from . import _lib, aggregate, capture, edge_mlp, padding as pad
from .aggregate import at_boundary, pna_aggregate
from .csr import tensor_version
from .linear import towers_compact_pays, towers_path_ok


def cached(owner, attr: str, extra, params, build):
    """``build()``, cached on ``owner.<attr>`` as ``(key, pack)`` with key = (``extra``, the in-place versions and the data
    pointers of ``params``, the parameters the pack reads).  The cache is neither read nor written inside a CUDA graph
    capture, where the packing is captured so that a replay follows the weights through optimizer steps, nor with autograd
    on and a parameter requiring grad, where the pack is part of the graph."""
    if capture.capturing() or (torch.is_grad_enabled() and any(p_.requires_grad for p_ in params)):
        return build()
    key = (extra, tuple(tensor_version(p_) for p_ in params), tuple(p_.data_ptr() for p_ in params))
    hit = getattr(owner, attr, None)
    if hit is not None and hit[0] == key:
        return hit[1]
    pack = build()
    setattr(owner, attr, (key, pack))
    return pack


def _stack(blocks, divide: bool):
    """Per-tower weight blocks over their output rows: block-diagonal when each tower reads only its own input columns."""
    return torch.block_diag(*blocks) if divide and len(blocks) > 1 else torch.cat(blocks, 0)


def first_layer_pack(lins, width: int, dst: int, src: int, divide: bool, fp: int | None = None, joined: bool = False):
    """The towers' first pre Linears ``lins`` for node-level GEMMs.  Each reads a destination block at columns
    [dst, dst + width), a source block at [src, src + width) and any edge columns after 2 * width.  Returns (W_dst, W_src,
    b, W_e): [T * fp, in] each (``_stack``), [T * fp], and the towers' edge columns stacked [T * width, edge] (None without
    edge columns).  ``fp`` pads every tower block with zero rows and zero bias entries, so the GEMM writes zero pad
    features.  ``joined`` returns (W_uv, b_uv) = ([W_dst; W_src], [0; b]) instead: U | V from one GEMM, no bias on U."""
    fp = fp or width
    halves = [[pad.expand_weight_rows(l.weight[:, c:c + width], width, fp) for l in lins] for c in (dst, src)]
    b = torch.cat([pad.pad_cols(l.bias, fp) for l in lins])
    if joined:
        w_uv = torch.cat([_stack(h, divide) for h in halves] if divide and len(lins) > 1 else halves[0] + halves[1], 0)
        return w_uv, torch.cat([torch.zeros_like(b), b])
    w_e = torch.cat([l.weight[:, 2 * width:] for l in lins], 0) if lins[0].weight.size(1) > 2 * width else None
    return _stack(halves[0], divide), _stack(halves[1], divide), b, w_e


def hidden_pack(lins):
    """The hidden pre Linears (``lins[t][k]``, k >= 1) as the message kernels take them: weights [L-1, T, F, F] and
    biases [L-1, T, F], empty with one Linear per tower."""
    L = len(lins[0])
    if L == 1:
        empty = lins[0][0].weight.new_empty(0)
        return empty, empty
    return (torch.stack([torch.stack([l[k].weight for l in lins]) for k in range(1, L)]),
            torch.stack([torch.stack([l[k].bias for l in lins]) for k in range(1, L)]))


class TowerLayer:
    """Mixed in next to ``nn.Module``; registers nothing.  The layer provides ``n_towers``, ``tower_in`` (the tower input
    width), ``avg`` (the scalers' degrees), ``_SRC_FIRST`` (the first pre Linear reads [src, dst, edge], not
    [dst, src, edge]), ``_AGG_FLAGS`` (extra ``pna_aggregate`` flags) and: ``_pre_linears()`` (each tower's pre Linears),
    ``_post_linears()`` (each tower's first post Linear), ``_affine(edge)``, ``_fused_layer_ok(edge, amp)`` (its own
    conditions on ``edge_messages``), ``_fused_messages(x, csr, edge, fp)`` (its ``edge_messages`` call on
    ``_message_operands``) and ``_torch_messages(x, csr, edge)`` (the [E, T * F] messages in slot order, in torch).
    The layer makes the kernel calls ``edge_messages`` and ``post_linear_towers_scaled`` itself, from its own module."""
    _SRC_FIRST = False
    _AGG_FLAGS = {}

    def _first_layer(self, fp=None, joined=False):
        F = self.tower_in
        lins = [l[0] for l in self._pre_linears()]
        return first_layer_pack(lins, F, F if self._SRC_FIRST else 0, 0 if self._SRC_FIRST else F, self.divide_input, fp,
                                joined)

    def _uv_weights(self, fp: int):
        lins = [l[0] for l in self._pre_linears()]
        return cached(self, "_uv_pack", fp, [p_ for l in lins for p_ in (l.weight, l.bias)],
                      lambda: self._first_layer(fp, joined=True))

    def _post_pack(self, fp: int):
        """The first post Linears as [T, F_out, (1 + S*A) * fp] (zero columns at the pad positions) and [T, F_out]."""
        lins = self._post_linears()
        blocks = 1 + len(self.aggregators) * len(self.scalers)
        return (torch.stack([pad.expand_weight_cols(l.weight, blocks, self.tower_in, fp) for l in lins]),
                torch.stack([l.bias for l in lins]))

    def _post_weights(self, fp: int):
        lins = self._post_linears()
        return cached(self, "_post_cache", fp, [p_ for l in lins for p_ in (l.weight, l.bias)], lambda: self._post_pack(fp))

    def _message_weights(self):
        """(W_dst, W_src, b1, W_e, W, bW): the pre Linears as ``edge_messages`` takes them."""
        lins = self._pre_linears()
        return cached(self, "_msg_pack", None, [p_ for l in lins for lin in l for p_ in (lin.weight, lin.bias)],
                      lambda: self._first_layer() + hidden_pack(lins))

    def _affine_terms(self, x, fp: int):
        """U = x W_dst^T, V = x W_src^T + b, both [N, T * fp]: the halves of one GEMM."""
        w_uv, b_uv = self._uv_weights(fp)
        uv = torch.addmm(b_uv, x, w_uv.t())
        half = uv.size(1) // 2
        return uv[:, :half], uv[:, half:]

    def _fused_messages_ok(self, x, edge, n_edges: int) -> bool:
        """The inputs ``edge_messages`` takes: float32 on the GPU and a tower width of at most 64 with more than one pre
        Linear; with autograd, graphs of at least ``edge_mlp.FUSED_TRAINING_MIN_EDGES`` edges (where the kernel path is
        faster).  Inside autocast the GEMMs make the operands, in the boundary dtype: the inputs' dtypes are not asked,
        the weights' is."""
        pre = self._pre_linears()[0]
        amp = aggregate.boundary_dtype() is not None
        return (edge_mlp.fused_step_pays(n_edges) and x.is_cuda and (amp or x.dtype == torch.float32)
                and pre[0].weight.dtype == torch.float32 and self._fused_layer_ok(edge, amp)
                and (len(pre) == 1 or self.tower_in <= _lib.EDGE_MLP_MAX_WIDTH))

    def _message_operands(self, x, csr, rows):
        """(A, Bm, b1, W, bW, C) for ``edge_messages``: A = x W_dst^T, Bm = x W_src^T, C = rows[perm] W_e^T for the
        per-edge ``rows`` the edge columns multiply (one GEMM for all towers; divide_input does not split them), the
        hidden Linears for the kernel."""
        W_dst, W_src, b1, W_e, W, bW = self._message_weights()
        C = None if W_e is None else at_boundary(rows.index_select(0, csr.perm.long()) @ W_e.t())
        return at_boundary(x @ W_dst.t()), at_boundary(x @ W_src.t()), b1, W, bW, C

    def _compact(self, x, fp: int) -> bool:
        """Compact post path: aggregate with the identity scaler only ([N, T * (1 + A) * fp]) and let
        ``post_linear_towers_scaled`` form the scaled copies in registers -- the [N, T * (1 + S*A) * fp] tensor is never
        written, nor saved for the backward.  Same arithmetic; float32 with more than one scaler, at the kernel's shapes,
        in training steps on graphs of at least ``linear.TOWERS_COMPACT_MIN_ROWS`` rows, where it measured faster."""
        lin = self._post_linears()[0]
        training = torch.is_grad_enabled() and any(p_.requires_grad for p_ in self.parameters())
        return (lin.weight.dtype == torch.float32 and lin.bias is not None
                and towers_path_ok(x, self.n_towers, fp, lin.out_features, len(self.scalers))
                and towers_compact_pays(x.size(0), training))

    def _tower_pitch(self, x) -> int:
        """The padded tower width in the kernels' dtype (bf16 pads to 8 columns)."""
        return pad.padded_width(self.tower_in, aggregate.boundary_dtype() or x.dtype)

    def _self_features(self, x, fp: int):
        if fp == self.tower_in:
            return x
        return pad.pad_blocks(x, self.n_towers, self.tower_in, fp) if self.divide_input else pad.pad_cols(x, fp)

    def _aggregate_towers(self, x, csr, edge, fp: int, x_self):
        """Every tower's messages and one aggregation: returns (the [N, T * (1 + S*A) * fp] aggregate, or with ``compact``
        the identity-scaled [N, T * (1 + A) * fp] one, compact)."""
        T = self.n_towers
        common = dict(towers=T, self_feat=x_self, self_divided=self.divide_input, **self._AGG_FLAGS)
        compact = self._compact(x, fp)
        scalers = ["identity"] if compact else self.scalers
        if self._affine(edge):
            U, V = (at_boundary(t) for t in self._affine_terms(x, fp))
            return pna_aggregate(V, csr, self.aggregators, scalers, self.avg, row_bias=U, **common), compact
        if self._fused_messages_ok(x, edge, csr.n_edges):
            msgs = self._fused_messages(x, csr, edge, fp)
        else:
            msgs = at_boundary(pad.pad_blocks(self._torch_messages(x, csr, edge), T, self.tower_in, fp))
        return pna_aggregate(msgs, csr, self.aggregators, scalers, self.avg, messages_in_csr_order=True, **common), compact
