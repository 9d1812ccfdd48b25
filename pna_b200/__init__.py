"""pna_b200 -- the PNA message-passing layer forward of lukecavabarrett/pna, rebuilt for H100 (sm_90a).

One hot path only (SURVEY.md section 8): destination-sorted CSR + one hand-written aggregation kernel
(gather, mean/max/min/std, degree scalers, concatenated output) behind the reference's own layer signatures.
The CUDA library is loaded lazily on first use and there is no CPU / PyTorch fallback for it.
"""
from ._lib import PnaError, build_library
from .capture import CaptureError
from .aggregate import aggregate_forward, avg_deg_from_histogram, pna_aggregate
from .csr import CSRGraph, build_csr, clear_csr_cache, csr_from_edge_index
from .pyg import PNAConv, PNAConvSimple
from .graph import Graph, avg_d_from_graphs, graph_csr
from .dgl_layers import PNALayer, PNASimpleLayer
from .static_batch import StaticBatch
from .set2set import S2SReadout, Set2Set
from . import capture, dense, padding, readout

__all__ = ["PnaError", "CaptureError", "build_library", "aggregate_forward", "avg_deg_from_histogram", "pna_aggregate", "CSRGraph",
           "build_csr", "clear_csr_cache", "csr_from_edge_index", "PNAConv", "PNAConvSimple", "Graph", "avg_d_from_graphs",
           "graph_csr", "PNALayer", "PNASimpleLayer", "StaticBatch", "Set2Set", "S2SReadout", "capture", "dense", "readout"]
__version__ = "0.1.0"
