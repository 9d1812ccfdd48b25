"""Oracles of the softmax / softmin / normalised_mean aggregators -- TEST INFRASTRUCTURE, imported only by tests/.

* ``dense_aggregate_softmax`` / ``_softmin`` / ``_normalised_mean`` / ``_identity``: the dense reference's functions
  (models/pytorch/pna/aggregators.py:10-14, 87-119) restated op for op in torch;
* ``weighted_rows``: the stable formulas on per-edge messages reduced by destination (rows without in-edges give 0),
  differentiable; in float64 it is the value the fp32 kernels are measured against;
* ``weighted``: the plain-C restatement in tests/weighted_oracle.c (the CUDA kernel's rounding order), compiled with gcc
  ``-ffp-contract=off`` into tests/emu/_build/ on first use.
"""
import ctypes as C
import os
import subprocess

import torch
from torch import Tensor

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "weighted_oracle.c")
LIB = os.path.join(HERE, "emu", "_build", "libweighted_oracle.so")
CODES = {"softmax": 9, "softmin": 10, "normalised_mean": 11}


def dense_aggregate_identity(X: Tensor, adj: Tensor, self_loop: bool = False) -> Tensor:
    """aggregators.py:10-14, op for op."""
    (_, N, N, _) = X.shape
    return torch.sum(torch.mul(X, torch.eye(N).reshape(1, N, N, 1)), dim=2)


def dense_aggregate_normalised_mean(X: Tensor, adj: Tensor, self_loop: bool = False) -> Tensor:
    """aggregators.py:87-99, op for op."""
    (B, N, N, _) = X.shape
    if self_loop:
        adj = adj + torch.eye(N).unsqueeze(0)
    rD = torch.mul(torch.pow(torch.sum(adj, -1, keepdim=True), -0.5), torch.eye(N).unsqueeze(0).repeat(B, 1, 1))
    adj = torch.matmul(torch.matmul(rD, adj), rD)
    return torch.sum(torch.mul(X, adj.unsqueeze(-1)), dim=2)


def dense_aggregate_softmax(X: Tensor, adj: Tensor, self_loop: bool = False) -> Tensor:
    """aggregators.py:102-114, op for op."""
    (B, N, N, Din) = X.shape
    if self_loop:
        adj = adj + torch.eye(N).unsqueeze(0)
    X_exp = torch.exp(X)
    adj = adj.unsqueeze(-1)
    X_exp = torch.mul(X_exp, adj)
    X_sum = torch.sum(X_exp, dim=2, keepdim=True)
    return torch.sum(torch.mul(torch.div(X_exp, X_sum), X), dim=2)


def dense_aggregate_softmin(X: Tensor, adj: Tensor, self_loop: bool = False) -> Tensor:
    """aggregators.py:117-119."""
    return -dense_aggregate_softmax(-X, adj, self_loop=self_loop)


DENSE = {"identity": dense_aggregate_identity, "normalised_mean": dense_aggregate_normalised_mean,
         "softmax": dense_aggregate_softmax, "softmin": dense_aggregate_softmin}


def in_degree(dst: Tensor, num_nodes: int, dtype=torch.float64) -> Tensor:
    return torch.zeros(num_nodes, dtype=dtype).index_add_(0, dst, torch.ones(dst.numel(), dtype=dtype))


def weights(dst: Tensor, wsrc: Tensor, num_nodes: int, dtype=torch.float64) -> Tensor:
    """normalised_mean's w_e = D_i^(-1/2) D_j^(-1/2) (i = dst, j = wsrc; 0 where a degree is 0 or j is not a row)."""
    deg = in_degree(dst, num_nodes, dtype)
    r = torch.where(deg > 0, deg.clamp(min=1).rsqrt(), torch.zeros_like(deg))
    ok = (wsrc >= 0) & (wsrc < num_nodes)
    rj = torch.where(ok, r[wsrc.clamp(0, num_nodes - 1)], torch.zeros((), dtype=dtype))
    return r[dst] * rj


def weighted_rows(msg: Tensor, dst: Tensor, num_nodes: int, name: str, wsrc: Tensor = None) -> Tensor:
    """The stable formulas on per-edge messages [E, F] reduced by destination (rows without in-edges give 0), in msg's
    dtype.  Differentiable."""
    F = msg.size(1)
    deg = in_degree(dst, num_nodes, msg.dtype)
    if name == "normalised_mean":
        return torch.zeros(num_nodes, F, dtype=msg.dtype).index_add(0, dst, msg * weights(dst, wsrc, num_nodes, msg.dtype)[:, None])
    sigma = -1.0 if name == "softmin" else 1.0
    n = sigma * msg
    M = torch.full((num_nodes, F), -float("inf"), dtype=msg.dtype).index_reduce(0, dst, n.detach(), "amax")
    e = torch.exp(n - M[dst])
    Z = torch.zeros(num_nodes, F, dtype=msg.dtype).index_add(0, dst, e)
    S = torch.zeros(num_nodes, F, dtype=msg.dtype).index_add(0, dst, e * n)
    y = sigma * S / torch.where(deg[:, None] > 0, Z, torch.ones_like(Z))
    return torch.where(deg[:, None] > 0, y, torch.zeros_like(y))


_lib = None


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or os.path.getmtime(LIB) < os.path.getmtime(SRC):
            os.makedirs(os.path.dirname(LIB), exist_ok=True)
            subprocess.run(["gcc", "-O2", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", LIB, SRC, "-lm"],
                           check=True)
        _lib = C.CDLL(LIB)
    return _lib


def weighted(msg: Tensor, dst: Tensor, n: int, name: str, wsrc: Tensor = None) -> Tensor:
    """y of the n destination rows (unscaled, [n, F]) in the CUDA kernel's rounding order.  msg: [E, F] per-edge messages
    in slot order; wsrc: the source node of every edge (normalised_mean's weight)."""
    msg = msg.contiguous().float()
    dst = dst.contiguous().long()
    wsrc = (dst if wsrc is None else wsrc).contiguous().long()
    out = torch.empty((n, msg.size(1)), dtype=torch.float32)
    rc = _load().pna_oracle_weighted(C.c_void_p(msg.data_ptr()), C.c_int64(n), C.c_int64(msg.size(1)), C.c_void_p(dst.data_ptr()),
                                     C.c_void_p(wsrc.data_ptr()), C.c_int64(dst.numel()), C.c_int32(CODES[name]),
                                     C.c_void_p(out.data_ptr()))
    if rc != 0:
        raise RuntimeError(f"pna_oracle_weighted failed: {rc}")
    return out
