"""Per-graph readouts of a batch of graphs on the aggregation kernel (SURVEY section 8(f)-4).

The reference nets finish with ``dgl.sum_nodes / mean_nodes / max_nodes(g, 'h')``
(realworld_benchmark/nets/*/pna_net.py:83-90) or ``global_mean_pool(x, batch)`` (models/pytorch_geometric/example.py:54):
a segmented reduction of node rows by graph id.  That is the aggregation path with "destination" = graph and
"source" = node, so it runs on ``pna_aggregate_fwd`` / ``pna_aggregate_bwd`` unchanged (graphs larger than the split
threshold become split rows); no separate kernel, no atomics, deterministic.  Empty graphs give zero rows.
Inside ``torch.autocast("cuda")`` an fp16 input (an autocast Linear's output) is upcast to fp32 at the kernel boundary;
fp32 and bf16 inputs are reduced in their own dtype (DESIGN section 2).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Optional

import torch

from . import capture
from .aggregate import at_boundary, pna_aggregate
from .csr import CSRGraph, build_csr, tensor_version
from .static_batch import StaticBatch, of_batch

_UNIT = {"log": 1.0, "lin": 1.0}        # identity scaler only: the averages are never read
_CACHE: "OrderedDict[tuple, tuple]" = OrderedDict()


def batch_csr(batch: torch.Tensor, n_graphs: int) -> CSRGraph:
    """CSR whose row g lists the nodes of graph g; cached on the identity of ``batch`` (one per mini-batch).  The ``batch``
    tensor of a ``StaticBatch`` is recognised by identity (``copy_`` bumps its version) and gets its padded readout CSR."""
    sb = of_batch(batch)
    if sb is not None:
        if int(n_graphs) != sb.max_graphs:
            raise ValueError(f"a StaticBatch's batch tensor reduces into its max_graphs = {sb.max_graphs} rows, not {n_graphs}")
        capture.pin(sb)
        return sb.readout_csr
    key = (batch.data_ptr(), tensor_version(batch), int(batch.numel()), int(n_graphs), str(batch.device))
    hit = _CACHE.get(key)
    if hit is not None:
        _CACHE.move_to_end(key)
        capture.pin(hit[1])
        return hit[1]
    n = int(batch.numel())
    csr = build_csr(torch.arange(n, device=batch.device), batch, n_graphs, n_src=n)
    csr.sources_unique = True       # one out-edge per node: the backward keeps its one-call path (aggregate.aggregate_backward)
    _CACHE[key] = (batch, csr)
    while len(_CACHE) > 8:
        _CACHE.popitem(last=False)
    return csr


def segment_reduce(x: torch.Tensor, batch: torch.Tensor, n_graphs: Optional[int] = None, reduce: str = "sum") -> torch.Tensor:
    """[N, F] node rows -> [n_graphs, F]; ``reduce`` in sum / mean / max / min.  Differentiable."""
    if reduce not in ("sum", "mean", "max", "min"):
        raise KeyError(reduce)
    if x.dim() != 2 or batch.dim() != 1 or batch.numel() != x.size(0):
        raise ValueError("x must be [N, F] and batch [N]")
    if n_graphs is None and of_batch(batch) is not None:
        n_graphs = of_batch(batch).max_graphs
    if n_graphs is None:
        capture.guard("a readout without its graph count (int(batch.max()) reads back)", "pass n_graphs / size")
        n_graphs = int(batch.max()) + 1 if batch.numel() else 0
    return pna_aggregate(at_boundary(x), batch_csr(batch, n_graphs), [reduce], ["identity"], _UNIT)


def global_add_pool(x: torch.Tensor, batch: torch.Tensor, size: Optional[int] = None) -> torch.Tensor:
    return segment_reduce(x, batch, size, "sum")


def global_mean_pool(x: torch.Tensor, batch: torch.Tensor, size: Optional[int] = None) -> torch.Tensor:
    return segment_reduce(x, batch, size, "mean")


def global_max_pool(x: torch.Tensor, batch: torch.Tensor, size: Optional[int] = None) -> torch.Tensor:
    return segment_reduce(x, batch, size, "max")


def _graph_batch(g, device) -> tuple:
    if isinstance(g, StaticBatch):       # padded nodes are in no graph, graph rows past the real count come out zero
        return g.batch, g.max_graphs
    sizes = getattr(g, "batch_num_nodes", None)
    sizes = sizes() if callable(sizes) else sizes
    sizes = torch.as_tensor(sizes, dtype=torch.long)
    cached = getattr(g, "_pna_b200_batch", None)
    if cached is None or cached.device != device:
        capture.guard("the node-to-graph index of this batched graph (a host-to-device copy)")
        cached = torch.repeat_interleave(torch.arange(sizes.numel()), sizes).to(device)
        try:
            g._pna_b200_batch = cached
        except Exception:
            pass
    return cached, int(sizes.numel())


def _nodes(g, feat: str, reduce: str) -> torch.Tensor:
    h = g.ndata[feat]
    batch, n_graphs = _graph_batch(g, h.device)
    return segment_reduce(h, batch, n_graphs, reduce)


def sum_nodes(g, feat: str) -> torch.Tensor:
    """dgl.sum_nodes(g, feat) for a batched graph exposing ``batch_num_nodes`` and ``ndata``."""
    return _nodes(g, feat, "sum")


def mean_nodes(g, feat: str) -> torch.Tensor:
    return _nodes(g, feat, "mean")


def max_nodes(g, feat: str) -> torch.Tensor:
    return _nodes(g, feat, "max")
