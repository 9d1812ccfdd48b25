"""PyG-signature PNA layers backed by the sm_90a aggregation kernel.

Drop-in for reference ``models/pytorch_geometric/pna.py``: same constructor arguments, same
``forward(x, edge_index, edge_attr=None)``, same parameter names (``pre_nns.{t}.{k}``, ``post_nns.{t}.{k}``,
``lin``, ``edge_encoder``; ``post_nn.{k}`` for the simple layer) so reference ``state_dict``s load unchanged.
torch_geometric is NOT needed: ``MessagePassing.propagate`` (gather + scatter) is what the kernel replaces.
``PNAConv`` shares its weight packs, messages and aggregation with the DGL ``PNALayer`` (towers.py).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
from torch import Tensor
from torch.nn import Linear, Module, ModuleList, ReLU, Sequential

from . import capture, padding as pad
from .aggregate import avg_deg_from_histogram, pna_aggregate, row_scales
from .edge_mlp import edge_messages
from .linear import compact_path_ok, linear_tf32x3, post_linear, post_linear_scaled, post_linear_towers_scaled
from .csr import CSRGraph, csr_from_edge_index
from .towers import TowerLayer, cached

_AGGRS = ("sum", "mean", "min", "max", "var", "std")          # aggregators.py:35-42
_SCALERS = ("identity", "amplification", "attenuation", "linear", "inverse_linear")  # scalers.py:32-38


def _reset(nn: Module) -> None:
    """torch_geometric.nn.inits.reset: call reset_parameters on every child that has one."""
    for m in nn.modules():
        if m is not nn and hasattr(m, "reset_parameters"):
            m.reset_parameters()


def _check_names(aggregators: List[str], scalers: List[str]) -> None:
    for a in aggregators:
        if a not in _AGGRS:
            raise KeyError(a)
    for s in scalers:
        if s not in _SCALERS:
            raise KeyError(s)


def _resolve_csr(x: Tensor, edge_index: Tensor, csr: Optional[CSRGraph]) -> CSRGraph:
    if csr is not None:
        if csr.n_nodes != x.size(0):
            raise ValueError("csr.n_nodes does not match x")
        return csr
    return csr_from_edge_index(edge_index, x.size(0))


class PNAConvSimple(Module):
    """reference pna.py:167-254.  message = x_j, aggregate = 4 aggregators x 3 scalers, update = post_nn."""

    def __init__(self, in_channels: int, out_channels: int, aggregators: List[str], scalers: List[str], deg: Tensor,
                 post_layers: int = 1, **kwargs):
        super().__init__()
        _check_names(aggregators, scalers)
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.aggregators = list(aggregators)
        self.scalers = list(scalers)
        self.F_in = in_channels
        self.F_out = out_channels
        self.avg_deg: Dict[str, float] = avg_deg_from_histogram(deg)          # pna.py:212-219

        width = len(aggregators) * len(scalers) * self.F_in                     # pna.py:221
        modules = [Linear(width, self.F_out)]
        for _ in range(post_layers - 1):
            modules += [ReLU(), Linear(self.F_out, self.F_out)]
        self.post_nn = Sequential(*modules)
        self.reset_parameters()

    def reset_parameters(self):
        _reset(self.post_nn)

    def aggregate_only(self, x: Tensor, edge_index: Optional[Tensor] = None, csr: Optional[CSRGraph] = None) -> Tensor:
        """The [N, S*A*F] tensor ``propagate`` returns in the reference (pna.py:236)."""
        csr = _resolve_csr(x, edge_index, csr)
        return pna_aggregate(x, csr, self.aggregators, self.scalers, self.avg_deg)

    def forward(self, x: Tensor, edge_index: Tensor, edge_attr: Optional[Tensor] = None, *,
                deg: Optional[Tensor] = None, csr: Optional[CSRGraph] = None) -> Tensor:
        # `deg` (precomputed in-degree) is accepted for signature compatibility with BASELINE.json's wording; the
        # in-degree always comes from the CSR row pointer, which is what degree(index) recounts in pna.py:247.
        agg, rs = self._aggregate_padded(x, _resolve_csr(x, edge_index, csr))
        return self._post(agg, rs, x.dtype)

    def _first_weight(self, dtype) -> Tensor:
        """weight of post_nn[0] at the padded feature width (zero columns at the pad positions)."""
        Fp = pad.padded_width(self.F_in, dtype)
        return pad.expand_weight_cols(self.post_nn[0].weight, len(self.aggregators) * len(self.scalers), self.F_in, Fp)

    def _compact(self, x: Tensor) -> bool:
        """Compact post path (SURVEY 8(f)-2): aggregate with the identity scaler only ([N, A*F]) and let the tensor-core
        linear regenerate the scaled copies in registers -- the [N, S*A*F] tensor is never written.  Same arithmetic."""
        Fp = pad.padded_width(self.F_in, x.dtype)
        lin0 = self.post_nn[0]
        return lin0.weight.dtype == torch.float32 and compact_path_ok(x, len(self.aggregators) * Fp, lin0.out_features,
                                                                      len(self.scalers))

    def _aggregate_padded(self, x: Tensor, csr: CSRGraph):
        """Aggregation at the kernel's 16-byte feature granularity: odd widths (e.g. 75) run on zero-padded rows.
        Returns (aggregate, row_scale): row_scale is None for the full [N, S*A*F] tensor, [N, S] for the compact one."""
        Fp = pad.padded_width(self.F_in, x.dtype)
        if self._compact(x):
            return (pna_aggregate(pad.pad_cols(x, Fp), csr, self.aggregators, ["identity"], self.avg_deg),
                    row_scales(csr, self.scalers, self.avg_deg))
        return pna_aggregate(pad.pad_cols(x, Fp), csr, self.aggregators, self.scalers, self.avg_deg), None

    def _post(self, agg: Tensor, row_scale: Optional[Tensor], dtype) -> Tensor:
        """post_nn on (a row block of) the aggregated tensor; padding is absorbed by zero columns of the first Linear."""
        lin0 = self.post_nn[0]
        # first Linear: tensor cores (3xTF32 wgmma, pna_linear_fwd) when the shape allows, else the library GEMM
        if row_scale is not None:
            out = post_linear_scaled(agg, row_scale, self._first_weight(dtype), lin0.bias)
        else:
            out = post_linear(agg, self._first_weight(dtype), lin0.bias)
        for m in list(self.post_nn)[1:]:
            out = m(out)
        return out

    @torch.no_grad()
    def forward_host(self, x: Tensor, edge_index: Tensor, out: Optional[Tensor] = None, row_blocks: int = 8) -> Tensor:
        """Inference entry point for HOST buffers (x, edge_index and the result live in pinned host memory), e.g. a
        CPU-resident caller of the reference's loops.  Same result as ``forward``; the PCIe transfers are overlapped with
        the device work instead of bracketing it:
          * edge_index goes up first and the CSR is built while x is still in flight on a copy stream;
          * after the aggregation, post_nn runs over row blocks and every finished block is copied back on a second
            copy stream while the next block is being computed.
        Returns the (pinned) host tensor; it is complete once the current stream has been synchronised."""
        dev = next(self.parameters()).device
        n = x.size(0)
        main = torch.cuda.current_stream(dev)
        if not hasattr(self, "_host_streams") or self._host_streams[0].device != dev:
            self._host_streams = (torch.cuda.Stream(device=dev), torch.cuda.Stream(device=dev))
        s_in, s_out = self._host_streams
        ei_d = edge_index.to(dev, non_blocking=True)
        s_in.wait_stream(main)
        with torch.cuda.stream(s_in):
            x_d = x.to(dev, non_blocking=True)
        csr = csr_from_edge_index(ei_d, n)                      # radix sort + views while x is on the wire
        main.wait_stream(s_in)
        x_d.record_stream(main)
        agg, rs = self._aggregate_padded(x_d, csr)
        if out is None:
            out = torch.empty((n, self.F_out), dtype=x.dtype, pin_memory=True)
        step = max(1, (n + row_blocks - 1) // row_blocks)
        for r0 in range(0, n, step):
            y = self._post(agg[r0:r0 + step], None if rs is None else rs[r0:r0 + step], x.dtype)
            s_out.wait_stream(main)
            with torch.cuda.stream(s_out):
                out[r0:r0 + step].copy_(y, non_blocking=True)
            y.record_stream(s_out)
        main.wait_stream(s_out)
        return out

    def __repr__(self):
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels})"


class PNAConv(TowerLayer, Module):
    """reference pna.py:17-164.  Towers, pre-MLP on [x_i || x_j (|| e)], aggregation, post-MLP on [x || agg], lin.

    With ``pre_layers == 1`` and no edge features the message is affine in (x_i, x_j):
    ``m = W_i x_i + W_j x_j + b`` (pna.py:94,147-149), so the E x F message tensor is never built: two node-level
    GEMMs give ``U = x W_i^T`` and ``V = x W_j^T + b`` and the kernel gathers V and adds U[i] per slot.  Otherwise
    (edge features or ``pre_layers > 1``) the messages are written once, in CSR slot order at the padded tower width, by
    ``pna_edge_msg_fwd`` (edge_mlp.py): the first pre Linear splits into the node GEMMs ``A = x W_i^T``,
    ``Bm = x W_j^T`` and one edge GEMM ``C = edge_encoder(edge_attr)[perm] W_e^T`` for all towers, and the kernel runs
    the rest of the pre-MLP per edge; the aggregation then reads them in slot order.  The messages are built in torch
    (the towers' ``pre_nns`` on gathered rows) only for inputs the kernel does not take: dtypes other than float32, and
    ``pre_layers > 1`` with a tower width ``F_in`` above 64 -- and for training steps on graphs below
    ``edge_mlp.FUSED_TRAINING_MIN_EDGES`` edges, where the torch path measured faster (launch overhead).

    Under ``torch.autocast("cuda")`` the operands of the kernels take ``aggregate.boundary_dtype()`` (DESIGN section 2):
    with bf16 the GEMM products U / V, A / Bm / C stay bf16 and run the bf16 aggregation, messages and compact tower
    post-linear, whatever x's dtype; with fp16 they are upcast to fp32 and run the fp32 kernels.  The tower width is padded
    for that dtype.  The weights stay fp32 throughout.
    """

    def __init__(self, in_channels: int, out_channels: int, aggregators: List[str], scalers: List[str], deg: Tensor,
                 edge_dim: Optional[int] = None, towers: int = 1, pre_layers: int = 1, post_layers: int = 1,
                 divide_input: bool = False, **kwargs):
        super().__init__()
        if divide_input:
            assert in_channels % towers == 0
        assert out_channels % towers == 0
        _check_names(aggregators, scalers)
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.aggregators = list(aggregators)
        self.scalers = list(scalers)
        self.edge_dim = edge_dim
        self.towers = towers
        self.divide_input = divide_input
        self.pre_layers = pre_layers
        self.F_in = in_channels // towers if divide_input else in_channels     # pna.py:76
        self.F_out = out_channels // towers                                     # pna.py:77
        self.avg_deg: Dict[str, float] = avg_deg_from_histogram(deg)            # pna.py:79-86

        if self.edge_dim is not None:
            self.edge_encoder = Linear(edge_dim, self.F_in)
        self.pre_nns = ModuleList()
        self.post_nns = ModuleList()
        for _ in range(towers):
            modules = [Linear((3 if edge_dim else 2) * self.F_in, self.F_in)]
            for _ in range(pre_layers - 1):
                modules += [ReLU(), Linear(self.F_in, self.F_in)]
            self.pre_nns.append(Sequential(*modules))
            width = (len(aggregators) * len(scalers) + 1) * self.F_in
            modules = [Linear(width, self.F_out)]
            for _ in range(post_layers - 1):
                modules += [ReLU(), Linear(self.F_out, self.F_out)]
            self.post_nns.append(Sequential(*modules))
        self.lin = Linear(out_channels, out_channels)
        self.reset_parameters()

    def reset_parameters(self):
        if self.edge_dim is not None:
            self.edge_encoder.reset_parameters()
        for nn in self.pre_nns:
            _reset(nn)
        for nn in self.post_nns:
            _reset(nn)
        self.lin.reset_parameters()

    n_towers = property(lambda self: self.towers)
    tower_in = property(lambda self: self.F_in)
    avg = property(lambda self: self.avg_deg)

    # -- what differs from the DGL layer on the shared tower path (towers.py) ------------------------------------------
    def _pre_linears(self):
        return [list(nn)[0::2] for nn in self.pre_nns]           # the Linears of each tower (ReLU between them)

    def _post_linears(self):
        return [nn[0] for nn in self.post_nns]

    def _affine(self, edge_attr) -> bool:
        return edge_attr is None and self.pre_layers == 1 and self.edge_dim is None

    def _fused_layer_ok(self, edge_attr, amp: bool) -> bool:
        return (edge_attr is None) == (self.edge_dim is None)

    def _prepared(self, Fp: int):
        """U|V and the first post Linears as one cached pack (``towers.cached``), w_uv, b_uv, w_post, b_post: every path of
        this layer that reads one reads the other.  U | V = x w_uv^T + b_uv is ONE node-level GEMM (pna.py:94,147-149), the
        first post Linear of every tower ONE batched GEMM or one tower kernel (pna.py:132)."""
        params = [p_ for nn in list(self.pre_nns) + list(self.post_nns) for p_ in nn[0].parameters()]
        return cached(self, "_prep", Fp, params, lambda: self._first_layer(Fp, joined=True) + self._post_pack(Fp))

    def _uv_weights(self, Fp: int):
        return self._prepared(Fp)[:2]

    def _post_weights(self, Fp: int):
        return self._prepared(Fp)[2:]

    def _fused_messages(self, x, csr, edge_attr, Fp: int):
        A, Bm, b1, W, bW, C = self._message_operands(x, csr, None if edge_attr is None else self.edge_encoder(edge_attr))
        return edge_messages(A, Bm, b1, W, bW, csr, self.towers, edge_term=C, pitch=Fp)

    def _torch_messages(self, x, csr, edge_attr):
        return self._messages_in_slot_order(x, csr, edge_attr)

    def _messages_in_slot_order(self, x: Tensor, csr: CSRGraph, edge_attr: Optional[Tensor]) -> Tensor:
        """General path (edge features or pre_layers > 1): pna.py:137-150 evaluated on CSR-ordered edges."""
        T, Fi = self.towers, self.F_in
        dst, src = csr.dst_of_slot, csr.col.long()
        xt = x.view(-1, T, Fi) if self.divide_input else x.view(-1, 1, Fi).expand(-1, T, -1)
        x_i, x_j = xt.index_select(0, dst), xt.index_select(0, src)
        if edge_attr is not None:
            e = self.edge_encoder(edge_attr).index_select(0, csr.perm.long())
            h = torch.cat([x_i, x_j, e.view(-1, 1, Fi).expand(-1, T, -1)], dim=-1)
        else:
            h = torch.cat([x_i, x_j], dim=-1)
        hs = [nn(h[:, t]) for t, nn in enumerate(self.pre_nns)]
        return torch.cat(hs, dim=1)

    # -- inference on the tensor cores: every GEMM of the layer through pna_linear_fwd (3xTF32, fp32-accurate) --------------
    def _tensor_core_pack(self, Fp: int):
        """Weights of the three dense steps at the shapes pna_linear_fwd takes (K a multiple of 32, 64/128/256 outputs), zero
        padded; cached per parameter version (``towers.cached``):
          U|V      [N, in -> K1] x [O1, K1]:  O1 >= 2*T*Fp rows (U block, V block, zero rows), bias only on the V block;
          towers   [N, T*W -> K2] x [O2, K2]: BLOCK-DIAGONAL -- output columns t*F_out.. read only tower t's W input
                   columns, so one launch does the first post Linear of every tower (pna.py:132) and its output is already
                   the concatenation torch.cat(outs, dim=1) of pna.py:134;
          lin      [N, O2] x [O3, O2]:        the final Linear (pna.py:135) on that buffer; pad columns meet zero weights."""
        params = [p_ for nn in list(self.pre_nns) + list(self.post_nns) for p_ in nn[0].parameters()] + list(self.lin.parameters())
        return cached(self, "_tc", ("tc", Fp), params, lambda: self._build_tensor_core_pack(Fp))

    def _build_tensor_core_pack(self, Fp: int):
        up32 = lambda v: (v + 31) // 32 * 32
        pick = lambda v: 64 if v <= 64 else 128 if v <= 128 else 256
        T, Fo = self.towers, self.F_out
        w_uv, b_uv, w_post, b_post = self._prepared(Fp)
        dev, dt = w_uv.device, w_uv.dtype
        K1, O1 = up32(w_uv.size(1)), pick(w_uv.size(0))
        w1 = torch.zeros((O1, K1), dtype=dt, device=dev); w1[: w_uv.size(0), : w_uv.size(1)] = w_uv
        b1 = torch.zeros(O1, dtype=dt, device=dev); b1[: b_uv.numel()] = b_uv
        W = w_post.size(2)                                          # (1 + S*A) * Fp columns per tower
        K2, O2 = up32(T * W), pick(T * Fo)
        w2 = torch.zeros((O2, K2), dtype=dt, device=dev)
        b2 = torch.zeros(O2, dtype=dt, device=dev)
        for t in range(T):
            w2[t * Fo:(t + 1) * Fo, t * W:(t + 1) * W] = w_post[t]
            b2[t * Fo:(t + 1) * Fo] = b_post[t]
        O3 = pick(self.out_channels)
        w3 = torch.zeros((O3, O2), dtype=dt, device=dev); w3[: self.out_channels, : T * Fo] = self.lin.weight
        b3 = torch.zeros(O3, dtype=dt, device=dev); b3[: self.out_channels] = self.lin.bias
        return dict(K1=K1, w1=w1, b1=b1, K2=K2, w2=w2, b2=b2, w3=w3, b3=b3)

    def _tensor_core_ok(self, x: Tensor, edge_attr, Fp: int) -> bool:
        import os
        T = self.towers
        return (x.is_cuda and x.dtype == torch.float32 and not torch.is_grad_enabled() and edge_attr is None and self.pre_layers == 1
                and self.edge_dim is None and len(self.post_nns[0]) == 1 and 2 * T * Fp <= 256 and T * self.F_out <= 256
                and self.out_channels <= 256 and x.size(0) > 0 and os.environ.get("PNA_B200_TENSOR_LINEAR", "1") != "0")

    def _forward_tensor_cores(self, x: Tensor, csr: CSRGraph, x_self: Tensor, Fp: int) -> Tensor:
        """No-grad forward with every dense step on the tensor cores (ZINC-shaped PNAConv(75,75,T=5): 1.73 -> see DESIGN.md);
        same arithmetic as the generic path up to fp32 summation order."""
        from .aggregate import aggregate_forward, output_width
        tc = self._tensor_core_pack(Fp)
        T, N = self.towers, x.size(0)
        uv = linear_tf32x3(pad.pad_cols(x, tc["K1"]), tc["w1"], tc["b1"])                       # [N, O1]: U | V | 0
        U, V = uv[:, : T * Fp], uv[:, T * Fp: 2 * T * Fp]
        # aggregation writes into a [N, K2] buffer whose pad columns are zero (allocated once per N: the kernel never
        # touches them), so the block-diagonal GEMM may read K2 columns
        width = T * output_width(Fp, len(self.aggregators), len(self.scalers), True)
        buf = getattr(self, "_tc_buf", None)
        if buf is None or buf.size(0) != N or buf.size(1) != tc["K2"] or buf.device != x.device:
            buf = torch.zeros((N, tc["K2"]), dtype=torch.float32, device=x.device)
            self._tc_buf = buf
        capture.pin(buf)           # a later call on another N replaces it
        aggregate_forward(V, csr, self.aggregators, self.scalers, self.avg_deg, towers=T, row_bias=U, self_feat=x_self,
                          self_divided=self.divide_input, out=buf[:, :width] if width < tc["K2"] else buf)
        h = linear_tf32x3(buf, tc["w2"], tc["b2"])                                               # [N, O2] = cat over towers | 0
        return linear_tf32x3(h, tc["w3"], tc["b3"])[:, : self.out_channels]

    def forward(self, x: Tensor, edge_index: Tensor, edge_attr: Optional[Tensor] = None, *,
                deg: Optional[Tensor] = None, csr: Optional[CSRGraph] = None) -> Tensor:
        csr = _resolve_csr(x, edge_index, csr)
        T = self.towers
        Fp = self._tower_pitch(x)
        x_self = self._self_features(x, Fp)
        if self._tensor_core_ok(x, edge_attr, Fp):
            return self._forward_tensor_cores(x, csr, x_self, Fp)
        out, compact = self._aggregate_towers(x, csr, edge_attr, Fp, x_self)
        if compact:
            # the first post Linear of every tower in one kernel, already the concatenation over the towers (pna.py:134)
            h = post_linear_towers_scaled(out, row_scales(csr, self.scalers, self.avg_deg), *self._post_weights(Fp))
            if len(self.post_nns[0]) > 1:
                Fo = self.F_out
                h = torch.cat([self._rest(nn, h[:, t * Fo:(t + 1) * Fo]) for t, nn in enumerate(self.post_nns)], dim=1)
            return self.lin(h)
        w_post, b_post = self._post_weights(Fp)
        out = out.view(x.size(0), T, -1)                       # [N, T, (1 + S*A) * Fp]  (pna.py:131)
        # first post Linear of all towers: one batched GEMM on the [N, T, W] view (tower = batch, no copy of the big tensor)
        h = torch.baddbmm(b_post.unsqueeze(1), out.transpose(0, 1), w_post.transpose(1, 2))      # [T, N, F_out]
        if len(self.post_nns[0]) > 1:
            h = torch.stack([self._rest(nn, h[t]) for t, nn in enumerate(self.post_nns)])
        out = h.transpose(0, 1).reshape(x.size(0), T * self.F_out) if T > 1 else h[0]
        return self.lin(out)

    @staticmethod
    def _rest(nn, h):
        for m in list(nn)[1:]:
            h = m(h)
        return h

    def __repr__(self):
        return f"{self.__class__.__name__}({self.in_channels}, {self.out_channels}, towers={self.towers})"
