"""``pna_aggregate``: the PNA neighbourhood aggregation as one call into libpna_sm90.so.

Replaces, for one layer call, the reference sequence (models/pytorch_geometric/pna.py:152-159 / :242-249):
``index_select`` of x_j, six ``scatter_add`` + ``scatter_min`` + ``scatter_max`` + ``degree`` passes over an
E x F message tensor (aggregators.py:9-32), three scaler passes (scalers.py:8-19) and three ``cat``s.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Mapping, Optional, Sequence, Union

import torch

from . import _lib, capture
from .csr import CSRGraph

_DTYPES = {torch.float32: _lib.PNA_F32, torch.bfloat16: _lib.PNA_BF16}
Names = Union[str, Sequence[str]]


def _names(v: Names) -> list:
    return v.split() if isinstance(v, str) else list(v)


def _ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _rows2d(t: torch.Tensor, what: str) -> torch.Tensor:
    if t.dim() != 2:
        raise ValueError(f"{what} must be 2-D, got shape {tuple(t.shape)}")
    if t.size(1) > 1 and t.stride(1) != 1:
        t = t.contiguous()
    if t.size(0) > 1 and t.stride(0) < t.size(1):
        t = t.contiguous()
    return t


def _padded(csr) -> bool:
    """Was ``csr`` built into fixed capacities (``CSRGraph.padded``)?  The aggregation takes any object with the CSR fields
    it reads, so one without the field is an ordinary CSR."""
    return getattr(csr, "padded", False)


HOT_SOURCE_FRACTION_FOR_L1 = 0.25      # CSRGraph.hot_source_fraction above which the gathers also allocate in L1


DYNAMIC_TAIL_MIN_PARTITION_COST = 256


def _dynamic_tail(csr: CSRGraph) -> bool:
    """Hand the last 30 % of the row partitions out dynamically (pna_agg_t.work_counter)?  Every grab restarts the warp's
    gather ring (serial latency: counter, partition bounds, first sources, first rows), so it pays only when a
    partition is much more work than that: the config-5 share (420 slots+12*rows per partition) gains, config 2 (49 per
    partition) loses."""
    return csr.n_part > 0 and (csr.n_edges + 12 * csr.n_nodes) / csr.n_part >= DYNAMIC_TAIL_MIN_PARTITION_COST


def _check_scaler_degree(t: torch.Tensor, n_rows: int, dev) -> torch.Tensor:
    if t.dtype not in (torch.int32, torch.float32) or t.device != dev or t.numel() != n_rows or not t.is_contiguous():
        raise ValueError("scaler_degree must be a contiguous int32 or float32 [n_rows] tensor on the same device")
    return t


def _check_degree_col(t: torch.Tensor, n_edges: int, dev) -> torch.Tensor:
    if t.dtype != torch.int32 or t.device != dev or t.numel() != n_edges or not t.is_contiguous():
        raise ValueError("degree_col must be a contiguous int32 [n_edges] tensor on the same device")
    return t


def _set_scaler_degree(d, t: torch.Tensor, n_rows: int, dev) -> None:
    """int32: pna_agg_t.scaler_degree.  float32 (a real-valued degree, the weighted dense adjacency) goes to the weighted
    entry points instead (:func:`_weights`)."""
    t = _check_scaler_degree(t, n_rows, dev)
    if t.dtype == torch.int32:
        d.scaler_degree = t.data_ptr()


# what a call with slot weights (or a float32 scaler degree) takes
ADJ_WEIGHT_AGGREGATORS = ("sum", "mean", "min", "max", "var", "std", "_skip")


def _weights(w: Optional[torch.Tensor], aggregators: Names, scaler_degree: Optional[torch.Tensor], n_edges: int, dev):
    """(slot_weight, scaler_degree_f) device pointers for pna_aggregate_*_weighted, or None when the call is unweighted.
    slot_weight: fp32 [E] in CSR slot order.  Weighted calls take the aggregators of ADJ_WEIGHT_AGGREGATORS only (the library
    returns PNA_ERR_UNSUPPORTED for the others; refused here before anything is enqueued)."""
    sdf = scaler_degree if scaler_degree is not None and scaler_degree.dtype == torch.float32 else None
    if w is None and sdf is None:
        return None
    bad = [a for a in _names(aggregators) if a not in ADJ_WEIGHT_AGGREGATORS]
    if bad:
        raise NotImplementedError(f"slot weights / a real-valued scaler degree take {ADJ_WEIGHT_AGGREGATORS[:-1]} only, "
                                  f"not {bad}")
    if w is not None and (w.dtype != torch.float32 or w.device != dev or w.numel() != n_edges or not w.is_contiguous()):
        raise ValueError("slot_weight must be a contiguous float32 [n_edges] tensor on the same device, in CSR slot order")
    return _ptr(w), _ptr(sdf)


def fold_finalize_enabled() -> bool:
    """PNA_B200_FOLD_FINALIZE=1: the warp that completes a split row also finalizes it (one launch per call)."""
    return os.environ.get("PNA_B200_FOLD_FINALIZE", "0") == "1"


def boundary_dtype() -> Optional[torch.dtype]:
    """The one rule for mixed precision (DESIGN section 2): the dtype in which the layers hand the products of their node
    and edge GEMMs to the kernels inside a CUDA ``torch.autocast`` region.

    * bf16 autocast: ``torch.bfloat16``.  U / V, A / Bm / C and the messages stay as autocast made them and go to the bf16
      kernel instances (aggregation, per-edge messages, compact tower post-linear); the weights stay fp32.
    * any other autocast dtype (float16): ``torch.float32``.  There are no fp16 kernel instances, so fp16 operands are
      upcast (``at_boundary``) and run the fp32 kernels.
    * no autocast: ``None`` -- the layers decide on the tensors' own dtypes, as they always have.
    Every layer asks this function (as ``aggregate.boundary_dtype()``), so it is the one place autocast is read."""
    if not torch.is_autocast_enabled("cuda"):
        return None
    return torch.bfloat16 if torch.get_autocast_dtype("cuda") == torch.bfloat16 else torch.float32


def at_boundary(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    """A kernel operand made inside an autocast region, at the kernel boundary: float16 is upcast to float32 (no fp16
    kernels); every other tensor, and every tensor outside autocast, passes as it is."""
    if t is not None and t.dtype == torch.float16 and boundary_dtype() is not None:
        return t.float()
    return t


def output_width(n_feat: int, n_aggr: int, n_scalers: int, has_self: bool) -> int:
    return (n_aggr * n_scalers + (1 if has_self else 0)) * n_feat


def aggregate_forward(gathered: torch.Tensor, csr: CSRGraph, aggregators: Names, scalers: Names,
                      avg_deg: Mapping[str, float], *, towers: int = 1, row_bias: Optional[torch.Tensor] = None,
                      self_feat: Optional[torch.Tensor] = None, self_divided: bool = True,
                      messages_in_csr_order: bool = False, zero_isolated: bool = False, relu_var: bool = False,
                      out: Optional[torch.Tensor] = None, row_ids: Optional[torch.Tensor] = None,
                      skip_light: bool = False, skip_hubs: bool = False, view=None, peer=None,
                      scaler_degree: Optional[torch.Tensor] = None, gather_l1: Optional[bool] = None,
                      degree_col: Optional[torch.Tensor] = None, slot_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Run the CUDA aggregation (no autograd).  Returns ``[N, towers * (has_self + S*A) * Ft]``.

    gathered : [n_src, F] rows that are gathered through ``csr.col`` (x for PNAConvSimple; V = x W_j^T + b for
               PNAConv), or -- with ``messages_in_csr_order`` -- [E, F] per-edge messages already in CSR slot order.
    row_bias : optional [N, F] destination-side term added to every gathered row of that destination.
    self_feat: optional node features copied to the front of every tower block of the output row
               (the ``torch.cat([x, out])`` of pna.py:131); ``self_divided`` tells whether tower t reads columns
               ``t*Ft:(t+1)*Ft`` (divide_input=True) or the same ``0:Ft`` (repeat, pna.py:126).
    degree_col: optional int32 [E]: for normalised_mean, the row of this CSR whose degree weighs each slot (in place of
               ``col``) -- what lets it run on messages in CSR order (pna_agg_t.degree_col).
    scaler_degree: optional [N] degree the scalers see: int32 (pna_agg_t.scaler_degree) or float32, a real-valued degree
               such as ``adj.sum(-1)`` of a weighted adjacency (pna_aggregate_fwd_weighted's scaler_degree_f).
    slot_weight: optional float32 [E] weight of every CSR slot (pna_aggregate_fwd_weighted): sum / mean / var / std weigh every
               message, min / max reduce over the slots of positive weight; a constant (no gradient).
    """
    if "normalised_mean" in _names(aggregators):
        # its weight D_i^(-1/2) D_j^(-1/2) reads the source's degree from the same CSR: every gathered row must be a row of
        # it, or degree_col names that row per slot
        if peer is not None or (degree_col is None and (messages_in_csr_order or gathered.size(0) != csr.n_nodes)):
            raise ValueError("normalised_mean needs gathered rows that are the CSR's own rows ([n_nodes, F], gathered through "
                             "col) or degree_col: not messages in CSR order without degree_col, a peer table, or a "
                             "[local ; halo] row buffer")
    if not gathered.is_cuda:
        raise ValueError("pna_b200 kernels run on CUDA tensors only; there is no CPU fallback")
    if gathered.dtype not in _DTYPES:
        raise TypeError(f"unsupported dtype {gathered.dtype}; libpna_sm90 takes float32 and bfloat16")
    dev = gathered.device
    if csr.device != dev:
        raise ValueError(f"CSR lives on {csr.device}, features on {dev}")
    gathered = _rows2d(gathered, "gathered")
    F = int(gathered.size(1))
    N = csr.n_nodes
    if F % towers != 0:
        raise ValueError(f"feature width {F} not divisible by towers={towers}")
    Ft = F // towers
    if messages_in_csr_order:
        if gathered.size(0) != csr.n_edges:
            raise ValueError("messages_in_csr_order needs one row per CSR slot")
    n_aggr, aggr_codes = _lib.pack_codes(aggregators, _lib.ALL_AGGR_CODES, "aggregator")
    n_scal, scal_codes = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
    if row_bias is not None:
        row_bias = _rows2d(row_bias.to(gathered.dtype), "row_bias")
        if tuple(row_bias.shape) != (N, F):
            raise ValueError(f"row_bias must be [{N}, {F}]")
    if self_feat is not None:
        self_feat = _rows2d(self_feat.to(gathered.dtype), "self_feat")
        need = F if self_divided else Ft
        if self_feat.size(0) != N or self_feat.size(1) != need:
            raise ValueError(f"self_feat must be [{N}, {need}]")
    width = towers * output_width(Ft, n_aggr, n_scal, self_feat is not None)
    if out is None:
        out = torch.empty((N, width), dtype=gathered.dtype, device=dev)
    else:
        if out.dtype != gathered.dtype or out.device != dev or out.dim() != 2 or out.size(0) != N or out.size(1) < width \
                or out.stride(1) != 1:
            raise ValueError("bad `out` buffer")
    if row_ids is not None:
        if row_ids.dtype != torch.int32 or not row_ids.is_contiguous() or row_ids.device != dev:
            raise ValueError("row_ids must be a contiguous int32 tensor on the same device")
    if gather_l1 is None:     # hot source rows (power-law graphs): keep gathered rows in L1 too (PNA_FLAG_GATHER_L1)
        gather_l1 = (not messages_in_csr_order) and peer is None and csr.hot_source_fraction > HOT_SOURCE_FRACTION_FOR_L1
    flags = (_lib.FLAG_GATHER_L1 if gather_l1 else 0) | \
            (_lib.FLAG_ZERO_ISOLATED if zero_isolated else 0) | (_lib.FLAG_SKIP_LIGHT if skip_light else 0) | \
            (_lib.FLAG_SKIP_HUBS if skip_hubs else 0) | (_lib.FLAG_RELU_VAR if relu_var else 0)
    partials = None if skip_hubs else csr.hub_partials(F)
    d = _lib.AggStruct(
        gathered=_ptr(gathered), ld_gathered=gathered.stride(0) if gathered.size(0) > 1 else F,
        rowptr=_ptr(csr.rowptr), col=None if messages_in_csr_order else (_ptr(csr.col) if csr.n_edges else None),
        row_bias=_ptr(row_bias), ld_row_bias=0 if row_bias is None else (row_bias.stride(0) if N > 1 else F),
        self_feat=_ptr(self_feat), ld_self=0 if self_feat is None else (self_feat.stride(0) if N > 1 else self_feat.size(1)),
        self_tower_stride=Ft if (self_feat is not None and self_divided) else 0,
        out=_ptr(out), ld_out=out.stride(0) if N > 1 else out.size(1),
        n_rows=N, n_feat=F, n_towers=towers, dtype=_DTYPES[gathered.dtype],
        n_aggr=n_aggr, aggr_codes=aggr_codes, n_scalers=n_scal, scaler_codes=scal_codes,
        avg_log=float(avg_deg["log"]), avg_lin=float(avg_deg.get("lin", 1.0)),
        flags=flags, split_threshold=csr.split_threshold, chunk_edges=csr.chunk_edges,
        hub_info=_ptr(csr.hub_info) if csr.n_hubs else None, chunk_items=_ptr(csr.chunk_items) if csr.n_hubs else None,
        n_hubs=csr.n_hubs, n_chunks=csr.n_chunks, hub_partials=_ptr(partials), max_degree=int(csr.max_degree),
        row_ids=_ptr(row_ids), n_row_ids=0 if row_ids is None else int(row_ids.numel()))
    if scaler_degree is not None:
        _set_scaler_degree(d, scaler_degree, N, dev)
    weights = _weights(slot_weight, aggregators, scaler_degree, csr.n_edges, dev)
    if degree_col is not None:
        d.degree_col = _check_degree_col(degree_col, csr.n_edges, dev).data_ptr()
    if view is None and row_ids is None and _dynamic_tail(csr):
        d.work_counter = _ptr(csr.work_counter())      # the whole graph in one launch: dynamic tail of the streamed kernel
    if view is None and row_ids is None:
        view = csr.full_view()
        if fold_finalize_enabled() and not skip_hubs and peer is None:
            d.hub_done = _ptr(csr.hub_done())      # split rows finalized inside the same launch
    if view is not None and row_ids is None and N > 0:
        # light view (whole graph: built with the CSR; row subset: CSRGraph.masked_view) -> streamed-gather kernel
        d.light_rowptr, d.light_deg, d.part, d.n_part = _ptr(view.light_rowptr), _ptr(view.light_deg), _ptr(view.part), view.n_part
        d.light_col = _ptr(view.light_col) if csr.n_edges else None
        d.n_view_rows = view.n_view_rows or N
    if peer is not None:
        # destination-partitioned multi-GPU graph: (int64 device tensor of per-rank row-buffer pointers, shift);
        # col entries are owner << shift | row and remote rows are gathered over NVLink inside the kernel
        ptr_table, shift = peer
        if ptr_table.dtype != torch.int64 or ptr_table.device != dev:
            raise ValueError("peer pointer table must be an int64 tensor on the same device")
        d.peer_gathered, d.peer_shift = ptr_table.data_ptr(), int(shift)
    capture.pin(csr, view, scaler_degree, degree_col, slot_weight)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        if weights is None:
            _lib.check(_lib.lib().pna_aggregate_fwd(C.byref(d), stream))
        else:
            _lib.check(_lib.lib().pna_aggregate_fwd_weighted(C.byref(d), *weights, stream))
    return out


def row_scales(csr: CSRGraph, scalers: Names, avg_deg: Mapping[str, float]) -> torch.Tensor:
    """[N, S] fp32: the factor of every degree scaler for every row (scalers.py:8-29), bit-identical to what the
    aggregation epilogue multiplies by.  Input of ``pna_linear_scaled_fwd``; cached on the CSR (a graph constant), except on
    a padded CSR, whose rows change with every ``StaticBatch.build()``: computed on every call there."""
    n_scal, codes = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
    key = (codes, n_scal, float(avg_deg["log"]), float(avg_deg.get("lin", 1.0)))
    cache = {} if _padded(csr) else csr.__dict__.setdefault("_row_scale_cache", {})
    hit = cache.get(key)
    if hit is not None:
        capture.pin(csr, hit)
        return hit
    dev = csr.device
    out = torch.empty((csr.n_nodes, n_scal), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_row_scales(_ptr(csr.rowptr), csr.n_nodes, n_scal, codes, key[2], key[3], _ptr(out),
                                             torch.cuda.current_stream(dev).cuda_stream))
    if len(cache) > 8:
        cache.clear()
    cache[key] = out
    capture.pin(csr, out)
    return out


# ---- autograd ----------------------------------------------------------------------------------------------------
def aggregate_backward(grad_out: torch.Tensor, gathered: torch.Tensor, csr: CSRGraph, aggregators: Names, scalers: Names,
                       avg_deg: Mapping[str, float], *, towers: int = 1, row_bias: Optional[torch.Tensor] = None,
                       has_self: bool = False, messages_in_csr_order: bool = False, need_bias_grad: bool = False,
                       relu_var: bool = False, scaler_degree: Optional[torch.Tensor] = None,
                       degree_col: Optional[torch.Tensor] = None, slot_weight: Optional[torch.Tensor] = None):
    """Gradient of the aggregation w.r.t. ``gathered`` (and ``row_bias``) through ``pna_aggregate_bwd`` (fp32 results)."""
    dev = gathered.device
    gathered = _rows2d(gathered, "gathered")
    F = int(gathered.size(1))
    N = csr.n_nodes
    capture.pin(csr, scaler_degree, degree_col, slot_weight)
    n_aggr, aggr_codes = _lib.pack_codes(aggregators, _lib.ALL_AGGR_CODES, "aggregator")
    n_scal, scal_codes = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
    grad_out = _rows2d(grad_out.to(gathered.dtype), "grad_out")
    if row_bias is not None:
        row_bias = _rows2d(row_bias.to(gathered.dtype), "row_bias")
    # a padded readout CSR has no slot-transposed CSR; every source row has at most one out-edge, so the atomic backward adds
    # once per element and is deterministic as it is
    deterministic = backward_mode() == "deterministic" and not (_padded(csr) and csr.sources_unique)
    # every element is written (per-slot stores, or the forward's sums per source row), except the padding slots of a
    # padded CSR when the messages are in CSR order: their gradient must be zero, not whatever the memory held
    if deterministic and csr.n_edges and not (_padded(csr) and messages_in_csr_order):
        gg = torch.empty((gathered.size(0), F), dtype=torch.float32, device=dev)
    else:
        gg = torch.zeros((gathered.size(0), F), dtype=torch.float32, device=dev)
    gb = torch.empty((N, F), dtype=torch.float32, device=dev) if need_bias_grad else None
    d = _lib.AggStruct(
        gathered=_ptr(gathered), ld_gathered=gathered.stride(0) if gathered.size(0) > 1 else F,
        rowptr=_ptr(csr.rowptr), col=None if messages_in_csr_order else (_ptr(csr.col) if csr.n_edges else None),
        row_bias=_ptr(row_bias), ld_row_bias=0 if row_bias is None else (row_bias.stride(0) if N > 1 else F),
        self_feat=1 if has_self else None,     # only its presence matters here: it shifts the grad_out columns
        n_rows=N, n_feat=F, n_towers=towers, dtype=_DTYPES[gathered.dtype],
        n_aggr=n_aggr, aggr_codes=aggr_codes, n_scalers=n_scal, scaler_codes=scal_codes,
        avg_log=float(avg_deg["log"]), avg_lin=float(avg_deg.get("lin", 1.0)),
        flags=_lib.FLAG_RELU_VAR if relu_var else 0,
        split_threshold=csr.split_threshold, chunk_edges=csr.chunk_edges,
        hub_info=_ptr(csr.hub_info) if csr.n_hubs else None, chunk_items=_ptr(csr.chunk_items) if csr.n_hubs else None,
        n_hubs=csr.n_hubs, n_chunks=csr.n_chunks)
    if scaler_degree is not None:
        _set_scaler_degree(d, scaler_degree, N, dev)
    weights = _weights(slot_weight, aggregators, scaler_degree, csr.n_edges, dev)
    if degree_col is not None:
        d.degree_col = _check_degree_col(degree_col, csr.n_edges, dev).data_ptr()
    scratch = None
    if csr.n_hubs:   # per-chunk statistics + per-split-row coefficients
        scratch = torch.empty(((csr.n_chunks + csr.n_hubs) * 6, F), dtype=torch.float32, device=dev)
        d.hub_partials = scratch.data_ptr()
    ld_go = grad_out.stride(0) if N > 1 else grad_out.size(1)
    if deterministic:
        _backward_deterministic(d, grad_out, ld_go, gathered, csr, gg, gb, messages_in_csr_order, weights)
        return gg, gb
    # moments, the weighted sums and slot weights have no coefficient form (their per-slot gradient is not c0 + c1 * m):
    # atomic path
    if messages_in_csr_order or csr.n_edges == 0 or csr.sources_unique or _padded(csr) or backward_mode() == "atomic" \
            or any(a in _lib.MOMENTS + _lib.WEIGHTED for a in _names(aggregators)) \
            or weights is not None \
            or 2 * _round_up(F, 4) > _lib.query(_lib.QUERY_MAX_FEATURES):
        with torch.cuda.device(dev):
            args = (grad_out.data_ptr(), ld_go, gg.data_ptr(), F, _ptr(gb), F, torch.cuda.current_stream(dev).cuda_stream)
            if weights is None:
                _lib.check(_lib.lib().pna_aggregate_bwd(C.byref(d), *args))
            else:
                _lib.check(_lib.lib().pna_aggregate_bwd_weighted(C.byref(d), *weights, *args))
        return gg, gb
    # shared source rows: coefficients per destination row -> their sums over the out-edges of every source row (the
    # forward kernels on the transposed graph) -> grad_gathered; the only atomics route min / max (one per row and feature)
    Fp = _round_up(F, 4)
    coef = torch.empty((N, 2 * Fp), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_aggregate_bwd_coef(C.byref(d), grad_out.data_ptr(), ld_go, coef.data_ptr(), 2 * Fp, Fp, gg.data_ptr(), F,
                                                     _ptr(gb), F, torch.cuda.current_stream(dev).cuda_stream))
    sums = aggregate_forward(coef, csr.transposed(gathered.size(0)), ["sum"], ["identity"], {"log": 1.0, "lin": 1.0})
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_aggregate_bwd_combine(sums.data_ptr(), sums.stride(0), Fp, _ptr(gathered),
                                                        gathered.stride(0) if gathered.size(0) > 1 else F, _DTYPES[gathered.dtype],
                                                        gg.data_ptr(), F, gathered.size(0), F, torch.cuda.current_stream(dev).cuda_stream))
    return gg, gb


def _round_up(n: int, m: int) -> int:
    return (n + m - 1) // m * m


# Bound on the fp32 per-slot gradients [E, slab] of the deterministic backward: wider rows are done in feature slabs.
DETERMINISTIC_SCRATCH_BYTES = 1 << 30


def deterministic_slab_width(n_edges: int, n_feat: int, align: int) -> int:
    """Feature columns per slab of the deterministic backward: all of them if ``E * F * 4`` bytes fit
    DETERMINISTIC_SCRATCH_BYTES, else the widest multiple of ``align`` (16 bytes of the element type) that does; never more
    than the forward kernel takes (PNA_QUERY_MAX_FEATURES), which sums the slab over the reversed edges."""
    max_f = _lib.query(_lib.QUERY_MAX_FEATURES) // align * align
    if n_edges * n_feat * 4 <= DETERMINISTIC_SCRATCH_BYTES and n_feat <= max_f:
        return n_feat
    w = DETERMINISTIC_SCRATCH_BYTES // (4 * max(n_edges, 1)) // align * align
    return max(align, min(w, max_f))


def _backward_deterministic(d, grad_out, ld_go, gathered, csr: CSRGraph, gg, gb, messages_in_csr_order: bool,
                            weights=None) -> None:
    """No floating-point atomics: per feature slab, (1) ``pna_aggregate_bwd_slots`` stores the gradient of every message in
    CSR slot order, (2) the forward kernel sums those rows over the slot-transposed CSR (ascending slot ids per source row)
    into the ``gg`` column slab.  Messages in CSR order need step 1 only: its output is their gradient."""
    dev = gathered.device
    F, E = gg.size(1), csr.n_edges
    L = _lib.lib()
    stream = torch.cuda.current_stream(dev).cuda_stream

    def slots(*args):          # pna_aggregate_bwd_slots, or its weighted form (slot_weight, scaler_degree_f)
        if weights is None:
            return L.pna_aggregate_bwd_slots(C.byref(d), *args)
        return L.pna_aggregate_bwd_slots_weighted(C.byref(d), *weights, *args)
    if messages_in_csr_order:
        gs = gg if E else torch.empty((1, F), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(slots(grad_out.data_ptr(), ld_go, 0, F, gs.data_ptr(), F, _ptr(gb), F, stream))
        return
    w = deterministic_slab_width(E, F, 16 // gathered.element_size())
    buf = torch.empty(max(E, 1) * w, dtype=torch.float32, device=dev)
    tcsr = csr.slot_transposed(gathered.size(0)) if E else None
    for f0 in range(0, F, w):
        fc = min(w, F - f0)
        gs = buf[:max(E, 1) * fc].view(max(E, 1), fc)
        with torch.cuda.device(dev):
            _lib.check(slots(grad_out.data_ptr(), ld_go, f0, fc, gs.data_ptr(), fc, _ptr(gb), F, stream))
        if E:
            aggregate_forward(gs, tcsr, ["sum"], ["identity"], {"log": 1.0, "lin": 1.0}, out=gg[:, f0:f0 + fc])


def backward_mode() -> str:
    """Which backward runs for gathered rows: "atomic" (default) = ``pna_aggregate_bwd``, one call, a vector atomic per edge and
    feature chunk; ``PNA_B200_BWD=coef`` = per-destination coefficient rows (``pna_aggregate_bwd_coef``), their sums over the
    transposed graph through the forward kernels, ``pna_aggregate_bwd_combine`` -- atomics only for min / max.  The
    coefficient path avoids the atomics that contend on hot source rows (power-law graphs), but regrouping sum_i (c0_i + c1_i x_j) into sum_i c0_i + x_j sum_i c1_i cancels badly where many rows have var ~ 0
    (2.6x the fp32 error of the per-edge evaluation on a power-law multigraph), so it stays opt-in.  Calls whose list contains a
    moment aggregator, softmax, softmin or normalised_mean take the atomic path under ``PNA_B200_BWD=coef``: their gradient is
    not c0 + c1 * m.
    Under ``torch.use_deterministic_algorithms(True)`` (``warn_only`` too) "deterministic", whatever PNA_B200_BWD says: per-slot
    gradients (``pna_aggregate_bwd_slots``) summed over the reversed edges by the forward kernel, no floating-point atomics,
    the same bits on every run."""
    if torch.are_deterministic_algorithms_enabled():
        return "deterministic"
    return "coef" if os.environ.get("PNA_B200_BWD", "atomic") == "coef" else "atomic"


class _PNAAggregate(torch.autograd.Function):
    @staticmethod
    def forward(ctx, gathered, row_bias, self_feat, csr, aggregators, scalers, avg_deg, towers, self_divided,
                messages_in_csr_order, zero_isolated, relu_var=False, scaler_degree=None, degree_col=None, slot_weight=None):
        out = aggregate_forward(gathered, csr, aggregators, scalers, avg_deg, towers=towers, row_bias=row_bias,
                                self_feat=self_feat, self_divided=self_divided,
                                messages_in_csr_order=messages_in_csr_order, zero_isolated=zero_isolated, relu_var=relu_var,
                                scaler_degree=scaler_degree, degree_col=degree_col, slot_weight=slot_weight)
        ctx.save_for_backward(gathered, row_bias, self_feat)
        ctx.meta = (csr, _names(aggregators), _names(scalers), dict(avg_deg), towers, self_divided, messages_in_csr_order,
                    relu_var, scaler_degree, degree_col, slot_weight)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        gathered, row_bias, self_feat = ctx.saved_tensors
        csr, aggregators, scalers, avg_deg, towers, self_divided, in_order, relu_var, scaler_degree, degree_col, slot_weight = \
            ctx.meta
        grad_g, grad_b = aggregate_backward(
            grad_out, gathered, csr, aggregators, scalers, avg_deg, towers=towers, row_bias=row_bias,
            has_self=self_feat is not None, messages_in_csr_order=in_order, need_bias_grad=ctx.needs_input_grad[1],
            relu_var=relu_var, scaler_degree=scaler_degree, degree_col=degree_col, slot_weight=slot_weight)
        gs = None
        if self_feat is not None and ctx.needs_input_grad[2]:
            # the self block of every tower is a plain copy: its gradient is the matching slice of grad_out
            N, F = csr.n_nodes, gathered.size(1)
            Ft = F // towers
            blk = grad_out.reshape(N, towers, -1)[:, :, :Ft]
            gs = (blk.reshape(N, F) if self_divided else blk.sum(1)).to(self_feat.dtype)
        return (grad_g.to(gathered.dtype) if ctx.needs_input_grad[0] else None,
                grad_b.to(row_bias.dtype) if (grad_b is not None) else None, gs,
                None, None, None, None, None, None, None, None, None, None, None, None)


def pna_aggregate(gathered: torch.Tensor, csr: CSRGraph, aggregators: Names, scalers: Names,
                  avg_deg: Mapping[str, float], *, towers: int = 1, row_bias: Optional[torch.Tensor] = None,
                  self_feat: Optional[torch.Tensor] = None, self_divided: bool = True,
                  messages_in_csr_order: bool = False, zero_isolated: bool = False, relu_var: bool = False,
                  scaler_degree: Optional[torch.Tensor] = None, degree_col: Optional[torch.Tensor] = None,
                  slot_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Differentiable PNA aggregation (forward = one libpna_sm90 call).  See :func:`aggregate_forward`.  ``slot_weight`` is a
    constant: a tensor that requires grad is refused (no gradient flows to it)."""
    if slot_weight is not None and slot_weight.requires_grad and torch.is_grad_enabled():
        raise ValueError("slot_weight gets no gradient: pass a tensor that does not require grad (e.g. weight.detach())")
    needs_grad = torch.is_grad_enabled() and any(
        t is not None and t.requires_grad for t in (gathered, row_bias, self_feat))
    if not needs_grad:
        return aggregate_forward(gathered, csr, aggregators, scalers, avg_deg, towers=towers, row_bias=row_bias,
                                 self_feat=self_feat, self_divided=self_divided,
                                 messages_in_csr_order=messages_in_csr_order, zero_isolated=zero_isolated, relu_var=relu_var,
                                 scaler_degree=scaler_degree, degree_col=degree_col, slot_weight=slot_weight)
    return _PNAAggregate.apply(gathered, row_bias, self_feat, csr, aggregators, scalers, avg_deg, towers, self_divided,
                               messages_in_csr_order, zero_isolated, relu_var, scaler_degree, degree_col, slot_weight)


def avg_deg_from_histogram(deg: torch.Tensor) -> dict:
    """The ``avg_deg`` dictionary of the PyG ctor, op for op (pna.py:79-86)."""
    deg = deg.to(torch.float)
    total_no_vertices = deg.sum()
    bin_degrees = torch.arange(len(deg), device=deg.device)
    return {
        "lin": ((bin_degrees * deg).sum() / total_no_vertices).item(),
        "log": (((bin_degrees + 1).log() * deg).sum() / total_no_vertices).item(),
        "exp": ((bin_degrees.exp() * deg).sum() / total_no_vertices).item(),
    }
