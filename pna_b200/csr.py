"""Destination-sorted CSR of a graph, built once per graph by ``pna_csr_build`` and reused by every layer.

The reference re-derives the segmentation on every ``aggregate`` call (torch_scatter by ``edge_index[1]``,
reference models/pytorch_geometric/pna.py:153,157).  Every layer of a net -- and every one of the N/2 repeated
layers of the multitask model (models/pytorch/gnn_framework.py:90-94) -- sees the same graph, so the CSR is cached
by graph identity.
"""
from __future__ import annotations

import ctypes as C
from collections import OrderedDict
from dataclasses import dataclass, field
from typing import Optional

import torch

from . import _lib, capture


@dataclass
class LightView:
    """Slots of a subset of the rows below the split threshold, compacted (see include/pna_b200.h pna_csr_light_view)."""
    light_rowptr: torch.Tensor    # int32 [N+1]
    light_deg: torch.Tensor       # int32 [N], -1 = row not in this view
    light_col: torch.Tensor       # int32 [E]
    part: torch.Tensor            # int32 [n_part+1]
    n_part: int
    n_view_rows: int = 0          # > n_nodes: the view ends with one pseudo-row per chunk of the split rows


@dataclass
class CSRGraph:
    """In-edges of every node, segmented by destination (stable in edge order)."""
    n_nodes: int
    n_edges: int
    rowptr: torch.Tensor          # int32 [N+1]
    col: torch.Tensor             # int32 [E]  source node of each slot
    perm: torch.Tensor            # int32 [E]  original edge id of each slot
    split_threshold: int
    chunk_edges: int
    hub_info: torch.Tensor        # int32 [n_hubs, 4]  row, first chunk, n chunks, in-degree
    chunk_items: torch.Tensor     # int32 [n_chunks, 2]
    n_hubs: int
    n_chunks: int
    max_degree: int
    # light view (rows below the split threshold, slots compacted) + equal-cost row partition for the streaming kernel
    light_rowptr: Optional[torch.Tensor] = None   # int32 [N+1]
    light_deg: Optional[torch.Tensor] = None      # int32 [N], -1 for split rows
    light_col: Optional[torch.Tensor] = None      # int32 [E] (first n_light_edges valid)
    part: Optional[torch.Tensor] = None           # int32 [n_part+1]
    n_part: int = 0
    n_light_edges: int = 0
    _partials: dict = field(default_factory=dict, repr=False)
    _deg: Optional[torch.Tensor] = field(default=None, repr=False)
    _dst: Optional[torch.Tensor] = field(default=None, repr=False)
    hot_source_fraction: float = 0.0      # pna_csr_t.hot_source_fraction: share of the gathers going to frequent sources
    sources_unique: bool = False          # every source row has at most one out-edge (readouts): the backward's atomics never collide
    # built by pna_csr_build_padded into fixed capacities (static_batch.StaticBatch): slots past rowptr[n_nodes] are padding,
    # no row is split, max_degree / n_light_edges are unknown on the host, and _deg / _dst are refilled in place by every
    # StaticBatch.build()
    padded: bool = False

    @property
    def device(self) -> torch.device:
        return self.rowptr.device

    @property
    def in_degree(self) -> torch.Tensor:
        """int32 [N] in-degree, duplicates included (= torch_geometric.utils.degree(edge_index[1], N))."""
        if self._deg is None:
            self._deg = self.rowptr[1:] - self.rowptr[:-1]
        return self._deg

    @property
    def dst_of_slot(self) -> torch.Tensor:
        """int64 [E] destination row of each CSR slot."""
        if self._dst is None:
            if self.padded:     # repeat_interleave leaves the tail past the real slots undefined
                raise ValueError("a padded CSR has dst_of_slot only as StaticBatch.build() refills it")
            self._dst = torch.repeat_interleave(
                torch.arange(self.n_nodes, device=self.device), self.in_degree.long(), output_size=self.n_edges)
        return self._dst

    def hub_partials(self, n_feat: int) -> Optional[torch.Tensor]:
        """fp32 scratch for the split rows, [n_chunks, 4, n_feat]; allocated once per width."""
        if self.n_hubs == 0:
            return None
        buf = self._partials.get(n_feat)
        if buf is None:
            buf = torch.empty((self.n_chunks, 4, n_feat), dtype=torch.float32, device=self.device)
            self._partials[n_feat] = buf
        return buf

    def hub_done(self) -> Optional[torch.Tensor]:
        """int32 [9 * n_hubs] completion counters of the folded finalize (pna_agg_t.hub_done): zero-initialised once,
        left zero by every call.  One set per CSR: calls that share a CSR must be stream-ordered (as for hub_partials)."""
        if self.n_hubs == 0:
            return None
        buf = self._partials.get("done")
        if buf is None:
            buf = torch.zeros(9 * self.n_hubs, dtype=torch.int32, device=self.device)
            self._partials["done"] = buf
        return buf

    def work_counter(self) -> torch.Tensor:
        """One int32 of scratch for the dynamic tail of the streamed kernel (pna_agg_t.work_counter); zeroed by the library
        before every launch.  One per CSR: calls that share a CSR must be stream-ordered (as for hub_partials)."""
        buf = self._partials.get("work")
        if buf is None:
            buf = torch.zeros(1, dtype=torch.int32, device=self.device)
            self._partials["work"] = buf
        return buf

    def transposed(self, n_src: int) -> "CSRGraph":
        """CSR of the reversed edges (rows = the ``n_src`` source rows, gathered from the destinations): what the backward
        sums its per-destination coefficient rows over (pna_aggregate_bwd_coef).  Built on first use, kept with the graph."""
        key = ("T", int(n_src))
        t = self._partials.get(key)
        if t is None:
            if self.padded:
                raise ValueError("a padded CSR has no transposed CSR: its backward takes the atomic or deterministic path")
            capture.guard("the transposed CSR of this graph (the coefficient backward)")
            t = build_csr(self.dst_of_slot, self.col.long(), int(n_src), n_src=self.n_nodes)
            self._partials[key] = t
        return t

    def slot_transposed(self, n_src: int) -> "CSRGraph":
        """CSR of the reversed edges whose slots are the forward CSR slot ids (rows = the ``n_src`` source rows, each row's slot
        ids in ascending order): what the deterministic backward sums its per-slot gradients over (pna_aggregate_bwd_slots).
        Built on first use, kept with the graph."""
        key = ("S", int(n_src))
        t = self._partials.get(key)
        if t is None:
            capture.guard("the slot-transposed CSR of this graph (the deterministic and edge-message backwards)")
            t = build_csr(torch.arange(self.n_edges, device=self.device), self.col.long(), int(n_src), n_src=self.n_edges)
            self._partials[key] = t
        return t

    def masked_view(self, row_mask: torch.Tensor) -> LightView:
        """Light view of the rows with ``row_mask != 0`` only (uint8/bool [N]); other rows are skipped by the kernel."""
        capture.guard("CSRGraph.masked_view (a light view is per-graph state)", "build the view before the capture")
        N, dev = self.n_nodes, self.device
        mask = row_mask.to(device=dev, dtype=torch.uint8).contiguous()
        if mask.numel() != N:
            raise ValueError("row_mask must have one entry per row")
        n_part = int(min(65536, max(1, N // 2)))
        lrp = torch.empty(N + 1, dtype=torch.int32, device=dev)
        ldeg = torch.empty(N, dtype=torch.int32, device=dev)
        lcol = torch.empty(max(self.n_edges, 1), dtype=torch.int32, device=dev)
        part = torch.empty(n_part + 1, dtype=torch.int32, device=dev)
        L = _lib.lib()
        with torch.cuda.device(dev):
            nb = C.c_size_t(0)
            _lib.check(L.pna_csr_light_view_workspace_bytes(N, C.byref(nb)))
            ws = torch.empty(max(int(nb.value), 256), dtype=torch.uint8, device=dev)
            _lib.check(L.pna_csr_light_view(self.rowptr.data_ptr(), self.col.data_ptr() if self.n_edges else None, N,
                                            self.split_threshold, mask.data_ptr() if N else None, n_part, lrp.data_ptr(),
                                            ldeg.data_ptr() if N else None, lcol.data_ptr(), part.data_ptr(), ws.data_ptr(),
                                            ws.numel(), torch.cuda.current_stream(dev).cuda_stream))
        return LightView(lrp, ldeg, lcol, part, n_part, N)

    def full_view(self) -> Optional[LightView]:
        if self.light_rowptr is None:
            return None
        return LightView(self.light_rowptr, self.light_deg, self.light_col, self.part, self.n_part, self.n_nodes + self.n_chunks)

    def degree_histogram(self) -> torch.Tensor:
        """Histogram of in-degrees (the ``deg`` ctor argument of PNAConv; reference example.py:21-25)."""
        return torch.bincount(self.in_degree.long(), minlength=self.max_degree + 1)


def build_csr(src: torch.Tensor, dst: torch.Tensor, n_nodes: int, split_threshold: Optional[int] = None,
              chunk_edges: Optional[int] = None, n_src: Optional[int] = None) -> CSRGraph:
    """Build the CSR on the GPU through the C ABI.  ``src[e] -> dst[e]``; int64 CUDA tensors.

    ``n_src`` (default ``n_nodes``): number of source rows when they differ from the destination rows -- the
    destination-partitioned multi-GPU path gathers from ``[local rows ; halo rows]``.

    Reads its counters back (one stream synchronisation), so inside a CUDA graph capture it raises
    ``capture.CaptureError`` instead (the graph's first eager step builds the CSR)."""
    capture.guard("build_csr (the CSR of a graph not seen before)")
    if not src.is_cuda or not dst.is_cuda:
        raise ValueError("pna_b200.build_csr needs CUDA tensors (there is no CPU path)")
    if src.dtype != torch.int64 or dst.dtype != torch.int64:
        src, dst = src.long(), dst.long()
    src = src.contiguous()
    dst = dst.contiguous()
    E = int(src.numel())
    if int(dst.numel()) != E:
        raise ValueError("src and dst differ in length")
    N = int(n_nodes)
    dev = src.device
    split = int(split_threshold) if split_threshold is not None else _lib.query(_lib.QUERY_DEFAULT_SPLIT)
    chunk = int(chunk_edges) if chunk_edges is not None else min(_lib.query(_lib.QUERY_DEFAULT_CHUNK), split)
    cap_hubs = E // split + 1
    cap_chunks = E // chunk + cap_hubs + 1
    with torch.cuda.device(dev):
        rowptr = torch.empty(N + 1, dtype=torch.int32, device=dev)
        col = torch.empty(E, dtype=torch.int32, device=dev)
        perm = torch.empty(E, dtype=torch.int32, device=dev)
        hub_info = torch.empty((cap_hubs, 4), dtype=torch.int32, device=dev)
        chunk_items = torch.empty((cap_chunks, 2), dtype=torch.int32, device=dev)
        n_part = int(min(65536, max(1, N // 2)))
        light_rowptr = torch.empty(N + cap_chunks + 1, dtype=torch.int32, device=dev)   # real rows + chunk pseudo-rows
        light_deg = torch.empty(N + cap_chunks, dtype=torch.int32, device=dev)
        light_col = torch.empty(E, dtype=torch.int32, device=dev)
        part = torch.empty(n_part + 1, dtype=torch.int32, device=dev)
        L = _lib.lib()
        nbytes = C.c_size_t(0)
        _lib.check(L.pna_csr_workspace_bytes(N, E, C.byref(nbytes)))
        ws = torch.empty(max(int(nbytes.value), 256), dtype=torch.uint8, device=dev)
        st = _lib.CsrStruct(
            n_nodes=N, n_edges=E, split_threshold=split, chunk_edges=chunk,
            rowptr=rowptr.data_ptr(), col=col.data_ptr() if E else None, perm=perm.data_ptr() if E else None,
            hub_info=hub_info.data_ptr(), chunk_items=chunk_items.data_ptr(), cap_hubs=cap_hubs, cap_chunks=cap_chunks,
            n_src_nodes=int(n_src) if n_src is not None else 0,
            n_part=n_part, light_rowptr=light_rowptr.data_ptr(), light_deg=light_deg.data_ptr(),
            light_col=light_col.data_ptr() if E else None, part=part.data_ptr())
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.pna_csr_build(src.data_ptr() if E else None, dst.data_ptr() if E else None, C.byref(st),
                                   ws.data_ptr(), ws.numel(), stream))
    nh, nc = int(st.n_hubs), int(st.n_chunks)
    return CSRGraph(n_nodes=N, n_edges=E, rowptr=rowptr, col=col, perm=perm, split_threshold=split, chunk_edges=chunk,
                    hub_info=hub_info[:nh].clone() if nh else hub_info[:0], chunk_items=chunk_items[:nc].clone() if nc else chunk_items[:0],
                    n_hubs=nh, n_chunks=nc, max_degree=int(st.max_degree), light_rowptr=light_rowptr, light_deg=light_deg,
                    light_col=light_col, part=part, n_part=n_part, n_light_edges=int(st.n_light_edges),
                    hot_source_fraction=float(st.hot_source_fraction))


# ---- cache by graph identity ---------------------------------------------------------------------------------
_CACHE: "OrderedDict[tuple, tuple]" = OrderedDict()
_CACHE_SIZE = 16


def tensor_version(t: torch.Tensor):
    """In-place version counter for cache keys; inference-mode tensors do not track one (reading ``_version`` raises), and
    cannot be modified in place outside inference mode either, so a constant stands in for it."""
    return None if t.is_inference() else t._version


def csr_from_edge_index(edge_index: torch.Tensor, n_nodes: int, cache: bool = True) -> CSRGraph:
    """CSR of a PyG ``edge_index`` (row 0 = source j, row 1 = target i; aggregation index = row 1).

    Cached on (storage pointer, in-place version counter, shape, N, device): a new batch is a new tensor, an
    in-place edit bumps ``_version``; the cache keeps a reference to the tensor so the pointer cannot be recycled.
    """
    if edge_index.dim() != 2 or edge_index.size(0) != 2:
        raise ValueError("edge_index must have shape [2, E]")
    key = (edge_index.data_ptr(), tensor_version(edge_index), tuple(edge_index.shape), tuple(edge_index.stride()), int(n_nodes),
           str(edge_index.device))
    if cache:
        hit = _CACHE.get(key)
        if hit is not None:
            _CACHE.move_to_end(key)
            capture.pin(hit[1])
            return hit[1]
    g = build_csr(edge_index[0], edge_index[1], n_nodes)
    if cache:
        _CACHE[key] = (edge_index, g)
        while len(_CACHE) > _CACHE_SIZE:
            _CACHE.popitem(last=False)
    return g


def clear_csr_cache() -> None:
    _CACHE.clear()
