"""Fixed-capacity mini-batches whose graph is rebuilt inside a captured training step (DESIGN section 8).

A captured step replays the same kernels on the same buffers.  Shuffled training brings a new graph every step, so the
graph itself has to become data in fixed buffers, and its CSRs have to be built by kernels that never read back.
``StaticBatch`` owns those buffers for batches of at most ``max_nodes`` nodes, ``max_edges`` edges and ``max_graphs``
graphs, and hides the padding format from every caller:

* ``copy_(...)``, outside the capture: checks the capacities on the host (``ValueError`` before anything is enqueued) and
  copies the batch in.  Edges past the real ones get ``dst = -1``, nodes past the real ones graph ``-1``, and the static
  node / edge feature tensors (``ndata`` / ``edata``) are zero past the real rows.  ``node_mask`` / ``graph_mask`` and
  ``counts`` (real nodes, edges, graphs) are device tensors.
* ``build()``, capture-legal, first thing in the captured step: the row CSR, its slot-transposed CSR and the readout CSR
  by ``pna_csr_build_padded``, and every derived tensor a layer reads (``in_degree``, ``dst_of_slot``) refilled in place.
  Padded CSRs do not cache row scales (``aggregate.row_scales``).
* ``batch_norm(bn, h)``: ``nn.BatchNorm1d`` over the real rows only.
* ``check()``, outside the capture: raises ``PnaError`` if a build met an endpoint outside its range.

The DGL layers take a ``StaticBatch`` as ``g``; ``PNAConv`` / ``PNAConvSimple`` take ``csr=sb.csr`` with ``sb.edge_index``;
the readouts take ``sum_nodes(sb, feat)`` or ``global_mean_pool(x, sb.batch, sb.max_graphs)``.  A padded CSR has no split
rows, so a row of high in-degree is reduced by one warp (DESIGN section 8).
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import Mapping, Optional

import torch
import torch.nn as nn

from . import _lib, capture
from .csr import CSRGraph

__all__ = ["StaticBatch", "masked_batch_norm"]

_BY_BATCH: "weakref.WeakValueDictionary[int, StaticBatch]" = weakref.WeakValueDictionary()


def of_batch(batch) -> Optional["StaticBatch"]:
    """The StaticBatch whose node-to-graph tensor is ``batch`` (by identity), or None."""
    sb = _BY_BATCH.get(id(batch))
    return sb if sb is not None and sb.batch is batch else None


def masked_batch_norm(bn: nn.BatchNorm1d, h: torch.Tensor, mask: torch.Tensor) -> torch.Tensor:
    """``bn(h)`` with the statistics of the rows where ``mask`` is set, in torch ops without a host read (capture-safe).
    Training: normalised by the biased variance, the running statistics updated with the unbiased one, ``momentum`` (or, when
    None, the cumulative average ``1 / num_batches_tracked``) as ``nn.BatchNorm1d`` does.  Eval: the running statistics.
    Rows outside the mask come out zero and get a zero gradient.  Inside a CUDA autocast region it computes in float32, as
    autocast runs ``batch_norm``."""
    if torch.is_autocast_enabled("cuda") and h.dtype in (torch.float16, torch.bfloat16):
        h = h.float()
    m = mask.to(h.dtype).unsqueeze(1)
    if bn.training or bn.running_mean is None:
        n = m.sum()
        mean = (h * m).sum(0) / n
        d = (h - mean) * m
        var = (d * d).sum(0) / n
        if bn.training and bn.track_running_stats and bn.running_mean is not None:
            with torch.no_grad():
                bn.num_batches_tracked.add_(1)
                f = bn.momentum if bn.momentum is not None else 1.0 / bn.num_batches_tracked
                bn.running_mean.mul_(1 - f).add_(mean.detach() * f)
                bn.running_var.mul_(1 - f).add_(var.detach() * (n / (n - 1)) * f)
        y = (h - mean) * torch.rsqrt(var + bn.eps)
    else:
        y = (h - bn.running_mean) * torch.rsqrt(bn.running_var + bn.eps)
    if bn.affine:
        y = y * bn.weight + bn.bias
    return y * m


class _PaddedBuild:
    """One padded CSR: its CSRGraph, the pna_csr_t that fills it, the workspace and the edge list it is built from."""

    def __init__(self, n_rows: int, n_slots: int, n_src: int, src: torch.Tensor, dst: torch.Tensor, status: torch.Tensor):
        dev = src.device
        split = max(n_slots + 1, 2)
        chunk = min(_lib.query(_lib.QUERY_DEFAULT_CHUNK), split)
        n_part = int(min(65536, max(1, n_rows // 2)))
        i32 = dict(dtype=torch.int32, device=dev)
        self.csr = CSRGraph(
            n_nodes=n_rows, n_edges=n_slots, rowptr=torch.zeros(n_rows + 1, **i32), col=torch.zeros(n_slots, **i32),
            perm=torch.zeros(n_slots, **i32), split_threshold=split, chunk_edges=chunk, hub_info=torch.zeros((0, 4), **i32),
            chunk_items=torch.zeros((0, 2), **i32), n_hubs=0, n_chunks=0, max_degree=0,
            light_rowptr=torch.zeros(n_rows + 1, **i32), light_deg=torch.zeros(n_rows, **i32),
            light_col=torch.zeros(max(n_slots, 1), **i32), part=torch.zeros(n_part + 1, **i32), n_part=n_part, padded=True)
        self.csr._deg = torch.zeros(n_rows, **i32)
        c = self.csr
        self.struct = _lib.CsrStruct(
            n_nodes=n_rows, n_edges=n_slots, split_threshold=split, chunk_edges=chunk, rowptr=c.rowptr.data_ptr(),
            col=c.col.data_ptr() if n_slots else None, perm=c.perm.data_ptr() if n_slots else None, n_src_nodes=n_src,
            n_part=n_part, light_rowptr=c.light_rowptr.data_ptr(), light_deg=c.light_deg.data_ptr() if n_rows else None,
            light_col=c.light_col.data_ptr(), part=c.part.data_ptr())
        nb = C.c_size_t(0)
        _lib.check(_lib.lib().pna_csr_padded_workspace_bytes(n_rows, n_slots, C.byref(nb)))
        self.ws = torch.empty(max(int(nb.value), 256), dtype=torch.uint8, device=dev)
        self.src, self.dst, self.status = src, dst, status

    def enqueue(self, stream) -> None:
        E = self.csr.n_edges
        _lib.check(_lib.lib().pna_csr_build_padded(self.src.data_ptr() if E else None, self.dst.data_ptr() if E else None,
                                                   C.byref(self.struct), self.status.data_ptr(), self.ws.data_ptr(),
                                                   self.ws.numel(), stream))
        torch.sub(self.csr.rowptr[1:], self.csr.rowptr[:-1], out=self.csr._deg)


class StaticBatch:
    """Device buffers for one mini-batch of at most ``max_nodes`` nodes, ``max_edges`` edges and ``max_graphs`` graphs."""

    def __init__(self, max_nodes: int, max_edges: int, max_graphs: int, device=None):
        if min(max_nodes, max_edges, max_graphs) < 1:
            raise ValueError("StaticBatch capacities must be at least 1")
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        if dev.type != "cuda":
            raise ValueError("StaticBatch lives on a CUDA device (there is no CPU path)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        N, E, G = int(max_nodes), int(max_edges), int(max_graphs)
        self.max_nodes, self.max_edges, self.max_graphs, self.device = N, E, G, dev
        i64 = dict(dtype=torch.int64, device=dev)
        with torch.cuda.device(dev):
            self.edge_index = torch.zeros((2, E), **i64)          # [src; dst], dst = -1 past the real edges
            self.edge_index[1].fill_(-1)
            self.src, self.dst = self.edge_index[0], self.edge_index[1]
            self.batch = torch.full((N,), -1, **i64)              # node -> graph, -1 past the real nodes
            self.node_mask = torch.zeros(N, dtype=torch.bool, device=dev)
            self.graph_mask = torch.zeros(G, dtype=torch.bool, device=dev)
            self.counts = torch.zeros(3, **i64)                   # real nodes, edges, graphs
            self.status = torch.zeros((3, 4), dtype=torch.int32, device=dev)   # per build: error bits, edges, max degree, 0
            self._node_ids = torch.arange(N, **i64)
            self._graph_ids = torch.arange(G, **i64)
            self._slot_ids = torch.arange(E, **i64)
            self._transpose_dst = torch.full((E,), -1, **i64)
            self._rows = _PaddedBuild(N, E, N, self.src, self.dst, self.status[0])
            self._slots = _PaddedBuild(N, E, E, self._slot_ids, self._transpose_dst, self.status[1])
            self._readout = _PaddedBuild(G, N, N, self._node_ids, self.batch, self.status[2])
        self.csr: CSRGraph = self._rows.csr
        self.csr._dst = torch.zeros(E, **i64)
        self.csr._partials[("S", N)] = self._slots.csr         # slot_transposed(max_nodes) is this one, never rebuilt
        self.readout_csr: CSRGraph = self._readout.csr
        self.readout_csr.sources_unique = True
        self.ndata: dict = {}
        self.edata: dict = {}
        self._inputs: dict = {}        # (kind, name) -> the static tensor copy_ writes
        self.n_nodes = self.n_edges = self.n_graphs = 0
        _BY_BATCH[id(self.batch)] = self

    # -- host side of a step -------------------------------------------------------------------------------------------
    def copy_(self, g=None, *, src=None, dst=None, batch_num_nodes=None, edge_index=None, batch=None,
              num_graphs: Optional[int] = None, ndata: Optional[Mapping] = None, edata: Optional[Mapping] = None):
        """Copy one batch in: a DGL-style batched graph ``g`` (``edges()``, ``batch_num_nodes``, its ``ndata`` / ``edata``
        unless given), or ``src`` / ``dst`` (or a PyG ``edge_index``) with ``batch_num_nodes`` or a node-to-graph ``batch``
        (and ``num_graphs``).  Every size is checked against the capacities before anything is enqueued.  Outside a
        capture only (``CaptureError`` inside one).  Returns ``self``."""
        capture.guard("StaticBatch.copy_ (the step's input copies)", "call copy_ before replaying the captured step")
        if g is not None:
            from .graph import graph_edges
            src, dst = graph_edges(g)
            batch_num_nodes = getattr(g, "batch_num_nodes", None)
            batch_num_nodes = batch_num_nodes() if callable(batch_num_nodes) else batch_num_nodes
            ndata = getattr(g, "ndata", {}) if ndata is None else ndata
            edata = getattr(g, "edata", {}) if edata is None else edata
        elif edge_index is not None:
            src, dst = edge_index[0], edge_index[1]
        if src is None or dst is None or src.numel() != dst.numel():
            raise ValueError("StaticBatch.copy_ needs a graph, src and dst of one length, or edge_index")
        E = int(src.numel())
        sizes = None
        if batch_num_nodes is not None:
            sizes = torch.as_tensor(batch_num_nodes, dtype=torch.long).cpu()
            n, G = int(sizes.sum()), int(sizes.numel())
        elif batch is not None:
            n = int(batch.numel())
            G = int(num_graphs) if num_graphs is not None else (int(batch.max()) + 1 if n else 0)
        else:
            raise ValueError("StaticBatch.copy_ needs batch_num_nodes, a batched graph or batch")
        for what, have, cap in (("max_nodes", n, self.max_nodes), ("max_edges", E, self.max_edges),
                                ("max_graphs", G, self.max_graphs)):
            if have > cap:
                raise ValueError(f"the batch exceeds {what}: {have} > {cap}")
        feats = [("ndata", k, v, n, self.max_nodes) for k, v in dict(ndata or {}).items()] + \
                [("edata", k, v, E, self.max_edges) for k, v in dict(edata or {}).items()]
        for kind, k, v, rows, cap in feats:
            if v.size(0) != rows:
                raise ValueError(f"{kind}[{k!r}] has {v.size(0)} rows, the batch {rows}")
            buf = self._inputs.get((kind, k))
            if buf is not None and (buf.shape[1:] != v.shape[1:] or buf.dtype != v.dtype):
                raise ValueError(f"{kind}[{k!r}] is {v.dtype} {tuple(v.shape[1:])} per row, the static tensor "
                                 f"{buf.dtype} {tuple(buf.shape[1:])}")

        self.src[:E].copy_(src)
        self.src[E:].zero_()
        self.dst[:E].copy_(dst)
        self.dst[E:].fill_(-1)
        if sizes is not None:
            batch = torch.repeat_interleave(torch.arange(G), sizes)
        self.batch[:n].copy_(batch)
        self.batch[n:].fill_(-1)
        torch.lt(self._node_ids, n, out=self.node_mask)
        torch.lt(self._graph_ids, G, out=self.graph_mask)
        for i, v in enumerate((n, E, G)):
            self.counts[i].fill_(v)
        for kind, k, v, rows, cap in feats:
            buf = self._inputs.get((kind, k))
            if buf is None:
                buf = torch.zeros((cap,) + tuple(v.shape[1:]), dtype=v.dtype, device=self.device)
                self._inputs[(kind, k)] = buf
            buf[:rows].copy_(v)
            buf[rows:].zero_()
            getattr(self, kind)[k] = buf      # the net may have replaced the entry: the static tensor comes back
        self.n_nodes, self.n_edges, self.n_graphs = n, E, G
        return self

    # -- device side of a step (capture-legal) -------------------------------------------------------------------------
    def build(self) -> "StaticBatch":
        """Enqueue the row CSR, the slot-transposed CSR and the readout CSR of the current batch, and refill ``in_degree``
        and ``dst_of_slot``.  Kernel launches, sorts and memsets only: legal inside a CUDA graph capture."""
        L = _lib.lib()
        with torch.cuda.device(self.device):
            st = torch.cuda.current_stream(self.device).cuda_stream
            self._rows.enqueue(st)
            _lib.check(L.pna_csr_slot_rows(self.csr.rowptr.data_ptr(), self.csr.col.data_ptr() if self.max_edges else None,
                                           self.max_nodes, self.max_edges, self._transpose_dst.data_ptr(),
                                           self.csr._dst.data_ptr(), st))
            self._slots.enqueue(st)
            self._readout.enqueue(st)
        capture.pin(self)
        return self

    def check(self) -> dict:
        """Read the status words (synchronises: outside a capture).  Raises ``PnaError`` if a build met an endpoint outside
        its range; returns the real edge count and the largest in-degree of the last build."""
        capture.guard("StaticBatch.check (reads the build status back)", "call check() outside the captured step")
        s = self.status.cpu()
        for i, what in enumerate(("edge list", "slot-transposed edge list", "node-to-graph index")):
            if int(s[i, 0]) & 1:
                raise _lib.PnaError(_lib.PNA_ERR_INDEX, f"StaticBatch.build: the {what} has an endpoint outside its range")
        return {"edges": int(s[0, 1]), "max_degree": int(s[0, 2])}

    def batch_norm(self, bn: nn.BatchNorm1d, h: torch.Tensor) -> torch.Tensor:
        """``bn(h)`` over the real node rows (:func:`masked_batch_norm`)."""
        return masked_batch_norm(bn, h, self.node_mask)
