"""Graph objects for the DGL-signature layers.

``dgl`` is not a dependency: the layers accept ANY object exposing ``edges()`` (or ``all_edges()``) returning
``(src, dst)`` and ``number_of_nodes()`` (or ``num_nodes()``) -- a real ``dgl.DGLGraph`` qualifies.  ``Graph`` below is
the minimal such object, with the ``ndata`` / ``edata`` dictionaries the reference nets write to
(realworld_benchmark/nets/*/pna_net.py:81).  The destination-sorted CSR is built once and cached on the graph object.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import capture
from .csr import CSRGraph, build_csr, tensor_version
from .static_batch import StaticBatch

_ATTR = "_pna_b200_csr"


class Graph:
    def __init__(self, src: torch.Tensor, dst: torch.Tensor, num_nodes: int, batch_num_nodes: Optional[list] = None):
        self._src, self._dst, self._n = src.long(), dst.long(), int(num_nodes)
        self.ndata, self.edata = {}, {}
        self.batch_num_nodes = batch_num_nodes if batch_num_nodes is not None else [self._n]

    def edges(self):
        return self._src, self._dst

    def number_of_nodes(self) -> int:
        return self._n

    def number_of_edges(self) -> int:
        return int(self._src.numel())

    def in_degrees(self) -> torch.Tensor:
        return torch.bincount(self._dst, minlength=self._n)

    def to(self, device):
        g = Graph(self._src.to(device), self._dst.to(device), self._n, self.batch_num_nodes)
        g.ndata = {k: v.to(device) for k, v in self.ndata.items()}
        g.edata = {k: v.to(device) for k, v in self.edata.items()}
        return g


def graph_edges(g):
    if hasattr(g, "edges") and callable(g.edges):
        out = g.edges()
    elif hasattr(g, "all_edges"):
        out = g.all_edges()
    else:
        raise TypeError(f"{type(g).__name__} exposes neither edges() nor all_edges()")
    return out[0], out[1]


def graph_num_nodes(g) -> int:
    for name in ("number_of_nodes", "num_nodes"):
        if hasattr(g, name):
            return int(getattr(g, name)())
    raise TypeError(f"{type(g).__name__} exposes neither number_of_nodes() nor num_nodes()")


def graph_csr(g, device: torch.device) -> CSRGraph:
    """CSR of the graph on `device`, built on first use and cached on the object.  A ``StaticBatch`` hands out its padded
    CSR (built by its ``build()``), with no cache lookup."""
    if isinstance(g, StaticBatch):
        if g.device != device:
            raise ValueError(f"the StaticBatch lives on {g.device}, the features on {device}")
        capture.pin(g)
        return g.csr
    src, dst = graph_edges(g)
    n = graph_num_nodes(g)
    # a graph mutated in place (add_edges / remove_edges / add_self_loop) hands out different edge tensors or counts:
    # the stamp of what the cached CSR was built from is compared on every call
    # (foreign graph types such as dgl.DGLGraph materialise fresh edge tensors on every edges() call, so only the counts
    # are comparable there; this package's Graph also stamps the tensors' identity and in-place version)
    stamp = (n, int(src.numel()))
    if isinstance(g, Graph):
        stamp += (src.data_ptr(), dst.data_ptr(), tensor_version(src), tensor_version(dst))
    hit = getattr(g, _ATTR, None)
    if hit is not None and hit[0] == stamp and hit[1].device == device:
        capture.pin(hit[1])
        return hit[1]
    csr = build_csr(src.to(device), dst.to(device), n)
    try:
        setattr(g, _ATTR, (stamp, csr, src, dst))     # the tensors are kept so their storage cannot be recycled
    except Exception:
        pass
    return csr


def avg_d_from_graphs(graphs) -> dict:
    """``avg_d`` of the real-world drivers (realworld_benchmark/main_molecules.py:368-372): statistics of the in-degrees
    of all training graphs."""
    D = torch.cat([torch.bincount(graph_edges(g)[1].cpu(), minlength=graph_num_nodes(g)).float() for g in graphs])
    return dict(lin=torch.mean(D).item(), exp=torch.mean(torch.exp(torch.div(1, D)) - 1).item(), log=torch.mean(torch.log(D + 1)).item())
