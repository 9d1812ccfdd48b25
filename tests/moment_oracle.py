"""Oracles of the moment aggregators -- TEST INFRASTRUCTURE, imported only by tests/.

* ``dense_aggregate_moment``: the dense reference's ``aggregate_moment`` (models/pytorch/pna/aggregators.py:122-134, with the
  ``aggregate_mean`` it calls, :17-27) restated op for op in torch;
* ``moment_rows``: the same formula on per-edge messages reduced by destination (PyG-style isolated rows), differentiable;
  in float64 it is the value the fp32 kernels are measured against;
* ``moment``: the plain-C restatement in tests/moment_oracle.c (the CUDA kernel's rounding order), compiled with gcc
  ``-ffp-contract=off`` into tests/emu/_build/ on first use.
"""
import ctypes as C
import os
import subprocess

import torch
from torch import Tensor

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "moment_oracle.c")
LIB = os.path.join(HERE, "emu", "_build", "libmoment_oracle.so")
EPS = 1e-5


def dense_aggregate_mean(X: Tensor, adj: Tensor, self_loop: bool = False) -> Tensor:
    """models/pytorch/pna/aggregators.py:17-27, op for op.  X [B, N, N, F], adj [B, N, N]."""
    if self_loop:
        (B, N, _) = adj.shape
        adj = adj + torch.eye(N, device=adj.device).unsqueeze(0)
    D = torch.sum(adj, -1, keepdim=True)
    X_sum = torch.sum(torch.mul(X, adj.unsqueeze(-1)), dim=2)
    return torch.div(X_sum, D)


def dense_aggregate_moment(X: Tensor, adj: Tensor, n: int, self_loop: bool = False) -> Tensor:
    """models/pytorch/pna/aggregators.py:122-134, op for op (self_loop=True adds I here AND in the mean, as there)."""
    if self_loop:
        (B, N, _) = adj.shape
        adj = adj + torch.eye(N, device=adj.device).unsqueeze(0)
    D = torch.sum(adj, -1, keepdim=True)
    X_mean = dense_aggregate_mean(X, adj, self_loop=self_loop)
    X_n = torch.div(torch.sum(torch.mul(torch.pow(X - X_mean.unsqueeze(2), n), adj.unsqueeze(-1)), dim=2), D)
    return torch.sign(X_n) * torch.pow(torch.abs(X_n) + EPS, 1. / n)


def moment_rows(msg: Tensor, dst: Tensor, num_nodes: int, k: int) -> Tensor:
    """The same formula on per-edge messages [E, F] reduced by destination (PyG-style: rows without in-edges give 0), in
    msg's dtype -- with float64 inputs the reference value the fp32 kernels are measured against.  Differentiable."""
    F = msg.size(1)
    deg = torch.zeros(num_nodes, dtype=msg.dtype).index_add_(0, dst, torch.ones(dst.numel(), dtype=msg.dtype))
    cnt = deg.clamp(min=1).unsqueeze(1)
    mu = torch.zeros(num_nodes, F, dtype=msg.dtype).index_add(0, dst, msg) / cnt
    M = torch.zeros(num_nodes, F, dtype=msg.dtype).index_add(0, dst, (msg - mu[dst]) ** k) / cnt
    r = torch.sign(M) * torch.pow(torch.abs(M) + EPS, 1.0 / k)
    return torch.where(deg.unsqueeze(1) > 0, r, torch.zeros_like(r))


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


def moment(x, edge_index, n, k):
    """r_k of the n destination rows (unscaled, [n, F]) in the CUDA kernel's rounding order.  x: [n_src, F] rows gathered
    through edge_index[0] (per-edge messages: edge_index[0] = arange(E))."""
    x = x.contiguous().float()
    src, dst = edge_index[0].contiguous().long(), edge_index[1].contiguous().long()
    out = torch.empty((n, x.size(1)), dtype=torch.float32)
    rc = _load().pna_oracle_moment(C.c_void_p(x.data_ptr()), C.c_int64(n), C.c_int64(x.size(1)), C.c_void_p(src.data_ptr()),
                                   C.c_void_p(dst.data_ptr()), C.c_int64(src.numel()), C.c_int32(k), C.c_void_p(out.data_ptr()))
    if rc != 0:
        raise RuntimeError(f"pna_oracle_moment failed: {rc}")
    return out
