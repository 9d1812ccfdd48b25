"""Synthetic workloads of BASELINE.json's configs (SURVEY.md section 8d).  CPU tensors, fixed seeds.

There is no network for ogbn-arxiv / ZINC / MNIST-superpixels, so each config is a synthetic graph of the stated shape;
the generators are deterministic so the CUDA path, the oracle and the reference arm all see identical inputs.
"""
from __future__ import annotations

import math
from typing import Tuple

import torch

ARXIV_NODES, ARXIV_EDGES = 169_343, 1_166_243   # ogbn-arxiv's node / edge counts


def degree_histogram(dst: torch.Tensor, n_nodes: int) -> torch.Tensor:
    """Histogram of in-degrees, the ``deg`` ctor argument (reference example.py:21-25)."""
    return torch.bincount(torch.bincount(dst, minlength=n_nodes))


def arxiv_like(n_nodes: int = ARXIV_NODES, n_edges: int = ARXIV_EDGES, n_feat: int = 128, seed: int = 0,
               skew: float = 3.0, dtype=torch.float32) -> Tuple[torch.Tensor, torch.Tensor]:
    """config 2: citation-graph-shaped CSR.  Sources uniform; destinations ``perm[floor(N * u**skew)]`` -- a heavy
    tail (max in-degree ~ E * N**(-1/skew), ~2e4 at the default size) and many in-degree-0 rows.  skew=1: uniform."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n_nodes, (n_edges,), generator=g)
    perm = torch.randperm(n_nodes, generator=g)
    u = torch.rand(n_edges, generator=g, dtype=torch.float64)
    dst = perm[(n_nodes * u.pow(skew)).long().clamp_(max=n_nodes - 1)]
    x = torch.randn(n_nodes, n_feat, generator=g).to(dtype)
    return torch.stack([src, dst]), x


def zinc_like(n_graphs: int = 12_000, n_feat: int = 75, seed: int = 0, dtype=torch.float32):
    """config 3: batched molecule-like graphs: nodes/graph ~ round(N(23.2, 4.3)) clipped to [9, 37], a random spanning
    tree plus ~8 % ring-closing edges, both directions; x = rows of a 28-entry embedding table (many identical
    neighbours -> zero-variance neighbourhoods, the adversarial case for std)."""
    g = torch.Generator().manual_seed(seed)
    sizes = torch.round(torch.randn(n_graphs, generator=g) * 4.3 + 23.2).clamp_(9, 37).long()
    offs = torch.cumsum(sizes, 0) - sizes
    n_nodes = int(sizes.sum())
    node_graph = torch.repeat_interleave(torch.arange(n_graphs), sizes)
    local = torch.arange(n_nodes) - offs[node_graph]
    # spanning tree: node k>0 of a graph attaches to a uniformly random earlier node of the same graph
    child = (local > 0).nonzero().flatten()
    parent = offs[node_graph[child]] + (torch.rand(child.numel(), generator=g) * local[child]).long()
    # ring closures: ~8 % extra edges between random node pairs of the same graph
    n_extra = int(0.08 * child.numel())
    gsel = torch.randint(0, n_graphs, (n_extra,), generator=g)
    a = offs[gsel] + (torch.rand(n_extra, generator=g) * sizes[gsel]).long()
    b = offs[gsel] + (torch.rand(n_extra, generator=g) * sizes[gsel]).long()
    keep = a != b
    u = torch.cat([child, a[keep]])
    v = torch.cat([parent, b[keep]])
    edge_index = torch.stack([torch.cat([u, v]), torch.cat([v, u])])
    table = torch.randn(28, n_feat, generator=g)
    atom = torch.randint(0, 28, (n_nodes,), generator=g)
    x = table[atom].to(dtype)
    return edge_index, x, node_graph


def superpixel_like(n_graphs: int = 15_000, nodes_per_graph: int = 70, k: int = 8, n_feat: int = 64, seed: int = 0,
                    dtype=torch.float32, chunk: int = 1000):
    """config 4 (per GPU): kNN graphs over random 2-D coordinates; every node sends an edge to each of its k nearest
    neighbours (reference realworld_benchmark/data/superpixels.py:56-75,142-148), so out-degree is k and in-degree
    varies (some 0)."""
    g = torch.Generator().manual_seed(seed)
    n = nodes_per_graph
    srcs, dsts = [], []
    for c0 in range(0, n_graphs, chunk):
        c = min(chunk, n_graphs - c0)
        pos = torch.rand(c, n, 2, generator=g)
        d = torch.cdist(pos, pos)
        d.diagonal(dim1=1, dim2=2).fill_(float("inf"))
        nbr = d.topk(k, dim=2, largest=False).indices                  # [c, n, k]
        base = (torch.arange(c0, c0 + c) * n).view(c, 1, 1)
        src = (torch.arange(n).view(1, n, 1).expand(c, n, k) + base).reshape(-1)
        dst = (nbr + base).reshape(-1)
        srcs.append(src)
        dsts.append(dst)
    edge_index = torch.stack([torch.cat(srcs), torch.cat(dsts)])
    x = torch.randn(n_graphs * n, n_feat, generator=g).to(dtype)
    return edge_index, x


def powerlaw(n_nodes: int = 1_250_000, n_edges: int = 12_500_000, n_feat: int = 256, seed: int = 0, alpha: float = 1.5,
             dtype=torch.float32, with_features: bool = True):
    """config 5 (one GPU's share by default): Zipf(alpha)-distributed source and destination ids over random
    permutations (inverse-CDF sampling of a bounded Pareto, so no rejection loop)."""
    g = torch.Generator().manual_seed(seed)

    def zipf_ids(n):
        u = torch.rand(n, generator=g, dtype=torch.float64)
        # bounded Pareto on [1, N+1) with tail exponent alpha-1  ->  rank ~ k^-alpha
        a = alpha - 1.0
        hi = float(n_nodes + 1)
        r = (1.0 - u * (1.0 - hi ** (-a))).pow(-1.0 / a)
        return (r.long() - 1).clamp_(0, n_nodes - 1)

    perm_s = torch.randperm(n_nodes, generator=g)
    perm_d = torch.randperm(n_nodes, generator=g)
    src = perm_s[zipf_ids(n_edges)]
    dst = perm_d[zipf_ids(n_edges)]
    x = torch.randn(n_nodes, n_feat, generator=g).to(dtype) if with_features else None
    return torch.stack([src, dst]), x


def multitask_like(n_graphs: int = 64, nodes_per_graph: int = 1000, n_feat: int = 16, seed: int = 1234):
    """config 1: block-diagonal batch of Erdos-Renyi graphs with a per-graph mean degree drawn from U[1, 32)
    (the reference's own generator, multitask_benchmark/datasets_generation/graph_generation.py:149-209, needs
    networkx + the reference tree, neither of which is on the GPU box); undirected, x ~ U[0,1)."""
    g = torch.Generator().manual_seed(seed)
    n = nodes_per_graph
    srcs, dsts = [], []
    for b in range(n_graphs):
        mean_deg = 1.0 + 31.0 * float(torch.rand(1, generator=g))
        m = int(mean_deg * n / 2)
        a = torch.randint(0, n, (m,), generator=g)
        c = torch.randint(0, n, (m,), generator=g)
        keep = a != c
        a, c = a[keep] + b * n, c[keep] + b * n
        srcs += [a, c]
        dsts += [c, a]
    edge_index = torch.stack([torch.cat(srcs), torch.cat(dsts)])
    x = torch.rand(n_graphs * n, n_feat, generator=g)
    return edge_index, x


def algorithmic_bytes(n_nodes: int, n_edges: int, n_feat: int, elem_size: int, n_out_cols: int) -> dict:
    """SURVEY.md section 8(d): compulsory traffic B_min and the no-reuse gather model B_gather, in bytes."""
    fixed = 4 * n_edges + 4 * (n_nodes + 1) + n_out_cols * n_nodes * elem_size
    return {"b_min": n_nodes * n_feat * elem_size + fixed, "b_gather": n_edges * n_feat * elem_size + fixed}


# ---- device-side generators for the multi-GPU configs (each rank generates only what it owns) -------------------------
def hash_features(ids: torch.Tensor, n_feat: int, dtype=torch.float32, chunk: int = 1 << 17) -> torch.Tensor:
    """x[r, j] = f(ids[r], j): a 32-bit integer mix mapped to [-1, 1) on a 2^-23 grid.  Integer arithmetic only, so the
    CPU (oracle) and every GPU rank produce bit-identical rows for any subset of node ids without communicating."""
    ids = ids.to(torch.int64)
    out = torch.empty((ids.numel(), n_feat), dtype=dtype, device=ids.device)
    j = torch.arange(n_feat, dtype=torch.int64, device=ids.device) * 0x85EBCA77
    for r0 in range(0, ids.numel(), chunk):
        h = (ids[r0:r0 + chunk, None] * 0x9E3779B1 + j[None, :] + 0x165667B1) & 0xFFFFFFFF
        h ^= h >> 15
        h = (h * 0x2C1B3C6D) & 0xFFFFFFFF
        h ^= h >> 12
        h = (h * 0x297A2D39) & 0xFFFFFFFF
        h ^= h >> 15
        out[r0:r0 + chunk] = ((h >> 8).to(torch.float32) * (2.0 ** -23) - 1.0).to(dtype)
    return out


def superpixel_shard(g0: int, n_graphs: int, device, nodes_per_graph: int = 70, k: int = 8, seed: int = 0, chunk: int = 2500):
    """config 4, graphs g0 .. g0+n_graphs-1 of the 60 000 (graph-batch shard of one rank), generated on `device`: kNN graphs
    over random 2-D coordinates, every node sends an edge to each of its k nearest neighbours
    (reference realworld_benchmark/data/superpixels.py:56-75,142-148).  One RNG stream per chunk of `chunk` graphs, so a
    graph does not depend on how many ranks share the batch.  Returns a LOCAL edge_index (node ids relative to g0)."""
    n = nodes_per_graph
    while n_graphs % chunk or g0 % chunk:
        chunk //= 2
        if chunk < 1:
            chunk = 1
            break
    srcs, dsts = [], []
    for c0 in range(g0, g0 + n_graphs, chunk):
        c = min(chunk, g0 + n_graphs - c0)
        g = torch.Generator(device=device).manual_seed(seed * 1_000_003 + c0)
        pos = torch.rand(c, n, 2, generator=g, device=device)
        d = torch.cdist(pos, pos)
        d.diagonal(dim1=1, dim2=2).fill_(float("inf"))
        nbr = d.topk(k, dim=2, largest=False).indices
        base = ((torch.arange(c0, c0 + c, device=device) - g0) * n).view(c, 1, 1)
        srcs.append((torch.arange(n, device=device).view(1, n, 1).expand(c, n, k) + base).reshape(-1))
        dsts.append((nbr + base).reshape(-1))
    return torch.stack([torch.cat(srcs), torch.cat(dsts)])


def powerlaw_stream(n_nodes: int, n_edges: int, device, seed: int = 0, alpha: float = 1.5, chunk: int = 12_500_000):
    """config 5 as a stream of edge chunks generated on `device` (every rank runs the same stream and keeps what it owns):
    Zipf(alpha) source and destination ids over random permutations, as :func:`powerlaw`.  Yields (src, dst) int64."""
    g = torch.Generator(device=device).manual_seed(seed)
    perm_s = torch.randperm(n_nodes, generator=g, device=device)
    perm_d = torch.randperm(n_nodes, generator=g, device=device)
    a = alpha - 1.0
    hi = float(n_nodes + 1)

    def zipf_ids(n):
        u = torch.rand(n, generator=g, dtype=torch.float64, device=device)
        r = (1.0 - u * (1.0 - hi ** (-a))).pow(-1.0 / a)
        return (r.long() - 1).clamp_(0, n_nodes - 1)

    for e0 in range(0, n_edges, chunk):
        c = min(chunk, n_edges - e0)
        yield perm_s[zipf_ids(c)], perm_d[zipf_ids(c)]


def sub_batch(edge_index: torch.Tensor, node_graph: torch.Tensor, graph_ids: torch.Tensor):
    """The mini-batch of graphs ``graph_ids`` (in that order) of a batched graph, as a shuffling data loader collates it:
    (edge_index renumbered from 0, batch_num_nodes, the node ids and the edge ids it took).  Edges are kept in their
    order within each graph."""
    n_graphs = int(node_graph.max()) + 1
    sizes = torch.bincount(node_graph, minlength=n_graphs)
    offs = torch.cumsum(sizes, 0) - sizes
    graph_ids = graph_ids.long()
    sub = sizes[graph_ids]
    node_ids = torch.repeat_interleave(offs[graph_ids] - (torch.cumsum(sub, 0) - sub), sub) + torch.arange(int(sub.sum()))
    new_id = torch.full((node_graph.numel(),), -1, dtype=torch.long)
    new_id[node_ids] = torch.arange(node_ids.numel())
    rank = torch.full((n_graphs,), -1, dtype=torch.long)
    rank[graph_ids] = torch.arange(graph_ids.numel())
    er = rank[node_graph[edge_index[1]]]
    eids = (er >= 0).nonzero().flatten()
    eids = eids[torch.sort(er[eids], stable=True).indices]
    return new_id[edge_index[:, eids]], sub, node_ids, eids
