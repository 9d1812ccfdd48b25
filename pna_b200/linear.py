"""First dense linear of the post-aggregation MLP on the H100 tensor cores (``pna_linear_fwd``, 3xTF32 wgmma).

``post_linear(a, weight, bias)`` is ``torch.nn.functional.linear`` for the shapes the kernel takes
(fp32, in_features % 32 == 0, out_features in {64, 128, 256}) and falls back to the library GEMM for every other shape --
the kernel is an accelerator for one GEMM shape family, not a requirement of the path.

``post_linear_scaled(a, row_scale, weight, bias)`` is the same linear fed by the COMPACT aggregate (SURVEY 8(f)-2):
``a`` is the ``[N, A*F]`` result of the identity scaler alone and the S scaled copies the reference concatenates
(pna.py:247-249) are regenerated in registers by the kernel's loaders -- ``linear(cat_s(row_scale[:, s:s+1] * a), W, b)``
without the ``[N, S*A*F]`` tensor ever being written or read.

Backward: the input gradient runs on the tensor cores (``pna_linear_bwd_data``, same accuracy, no atomics; the compact one
never forms the scaled copies).  The weight gradient stays a library fp32 GEMM (``library_grad_weight``): at config 2 on
H100 cuBLAS is faster than the tensor-core ``pna_linear_bwd_weight`` (DESIGN section 5), which ``linear_bwd_tf32x3``
still exposes.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _lib

_OUT_OK = (64, 128, 256)


def kernel_applies(a: torch.Tensor, weight: torch.Tensor) -> bool:
    if os.environ.get("PNA_B200_TENSOR_LINEAR", "1") == "0":       # opt out: keep the library fp32 GEMM
        return False
    return (a.is_cuda and a.dtype == torch.float32 and weight.dtype == torch.float32 and a.dim() == 2 and a.size(0) > 0
            and a.size(1) % 32 == 0 and weight.size(0) in _OUT_OK and a.stride(1) == 1 and a.stride(0) % 4 == 0
            and a.data_ptr() % 16 == 0)


def linear_tf32x3(a: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """y = a @ weight.T + bias through the C ABI (no autograd)."""
    n, k = a.shape
    o = weight.size(0)
    dev = a.device
    w = weight.detach().contiguous()
    b = None if bias is None else bias.detach().contiguous()
    y = torch.empty((n, o), dtype=torch.float32, device=dev)
    ws = torch.empty(2 * k * o, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_linear_fwd(a.data_ptr(), a.stride(0), w.data_ptr(), None if b is None else b.data_ptr(), y.data_ptr(),
                                             y.stride(0), n, k, o, ws.data_ptr(), ws.numel() * 4,
                                             torch.cuda.current_stream(dev).cuda_stream))
    return y


def linear_bwd_tf32x3(gy: torch.Tensor, a: torch.Tensor, row_scale: Optional[torch.Tensor], weight: torch.Tensor,
                      need_a: bool = True, need_w: bool = True):
    """(grad a, grad weight) of ``linear_tf32x3`` (row_scale None) or ``linear_scaled_tf32x3`` through the C ABI (no
    autograd); a gradient that is not needed is not computed and comes back as None."""
    if not (need_a or need_w):
        return None, None
    n, ka = a.shape
    o, k = weight.shape
    s = 1 if row_scale is None else row_scale.size(1)
    dev = a.device
    if not gy.is_contiguous() or gy.data_ptr() % 16:
        gy = gy.clone(memory_format=torch.contiguous_format)
    w = weight.detach().contiguous()
    rs = None if row_scale is None else row_scale.data_ptr()
    ga = torch.empty((n, ka), dtype=torch.float32, device=dev) if need_a else None
    gw = torch.empty((o, k), dtype=torch.float32, device=dev) if need_w else None
    L = _lib.lib()
    nb = C.c_size_t(0)
    _lib.check(L.pna_linear_bwd_workspace_bytes(n, k, o, s, C.byref(nb)))
    ws = torch.empty((nb.value + 3) // 4, dtype=torch.float32, device=dev)        # one buffer for both calls (stream order)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream(dev).cuda_stream
        if ga is not None:
            _lib.check(L.pna_linear_bwd_data(gy.data_ptr(), gy.stride(0), rs, s, w.data_ptr(), ga.data_ptr(), ga.stride(0), n, k, o,
                                             ws.data_ptr(), nb.value, st))
        if gw is not None:
            _lib.check(L.pna_linear_bwd_weight(gy.data_ptr(), gy.stride(0), a.data_ptr(), a.stride(0), rs, s, gw.data_ptr(), n, k, o,
                                               ws.data_ptr(), nb.value, st))
    return ga, gw


def library_grad_weight(gy: torch.Tensor, a: torch.Tensor, row_scale: Optional[torch.Tensor], weight: torch.Tensor) -> torch.Tensor:
    """grad weight of ``linear_tf32x3`` / ``linear_scaled_tf32x3`` as library fp32 GEMMs (cuBLAS: deterministic with a fixed
    workspace, as torch.use_deterministic_algorithms requires); with row scales one scaler block at a time, each
    ``fl(c_s * a)`` a temporary of a's size."""
    if row_scale is None:
        return gy.t() @ a
    ka = a.size(1)
    gw = torch.empty_like(weight)
    for s in range(row_scale.size(1)):
        torch.mm(gy.t(), a * row_scale[:, s:s + 1], out=gw[:, s * ka:(s + 1) * ka])
    return gw


class _Linear3xTF32(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, weight, bias):
        ctx.save_for_backward(a, weight)
        ctx.has_bias = bias is not None
        return linear_tf32x3(a, weight, bias)

    @staticmethod
    def backward(ctx, gy):
        a, weight = ctx.saved_tensors
        ga, _ = linear_bwd_tf32x3(gy, a, None, weight, ctx.needs_input_grad[0], False)
        gw = library_grad_weight(gy, a, None, weight) if ctx.needs_input_grad[1] else None
        gb = gy.sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None
        return ga, gw, gb


def post_linear(a: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    if not kernel_applies(a, weight):
        return torch.nn.functional.linear(a, weight, bias)
    if torch.is_grad_enabled() and (a.requires_grad or weight.requires_grad or (bias is not None and bias.requires_grad)):
        return _Linear3xTF32.apply(a, weight, bias)
    return linear_tf32x3(a, weight, bias)


# ---- compact path: a = identity-scaled aggregate [N, A*F], the S scaled copies exist only inside the kernel ----------


def compact_path_ok(x: torch.Tensor, n_a: int, n_out: int, n_scalers: int) -> bool:
    """Shape-level decision the layers take BEFORE aggregating: would a fresh fp32 [N, n_a] aggregate on x's device,
    with a [n_out, n_scalers * n_a] first post Linear, go through pna_linear_scaled_fwd?"""
    return (n_scalers > 1 and x.is_cuda and x.dtype == torch.float32 and x.size(0) > 0 and n_a % 32 == 0 and n_out in _OUT_OK
            and os.environ.get("PNA_B200_TENSOR_LINEAR", "1") != "0" and os.environ.get("PNA_B200_COMPACT_POST", "1") != "0")


def scaled_kernel_applies(a: torch.Tensor, weight: torch.Tensor, n_scalers: int) -> bool:
    return (n_scalers > 1 and kernel_applies(a, weight) and weight.size(1) == n_scalers * a.size(1)
            and os.environ.get("PNA_B200_COMPACT_POST", "1") != "0")


def linear_scaled_tf32x3(a: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor,
                         bias: Optional[torch.Tensor]) -> torch.Tensor:
    """y = cat_s(row_scale[:, s, None] * a) @ weight.T + bias through the C ABI (no autograd)."""
    n, ka = a.shape
    o, k = weight.shape
    s = row_scale.size(1)
    if k != s * ka or row_scale.size(0) != n or row_scale.dtype != torch.float32 or not row_scale.is_contiguous():
        raise ValueError("row_scale must be a contiguous fp32 [N, S] tensor and weight [O, S * a.size(1)]")
    dev = a.device
    w = weight.detach().contiguous()
    b = None if bias is None else bias.detach().contiguous()
    y = torch.empty((n, o), dtype=torch.float32, device=dev)
    ws = torch.empty(2 * k * o, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_linear_scaled_fwd(a.data_ptr(), a.stride(0), row_scale.data_ptr(), s, w.data_ptr(),
                                                    None if b is None else b.data_ptr(), y.data_ptr(), y.stride(0), n, k, o,
                                                    ws.data_ptr(), ws.numel() * 4, torch.cuda.current_stream(dev).cuda_stream))
    return y


class _LinearScaled3xTF32(torch.autograd.Function):
    """The scale factors are constants of the graph: no gradient for row_scale."""

    @staticmethod
    def forward(ctx, a, row_scale, weight, bias):
        ctx.save_for_backward(a, row_scale, weight)
        ctx.has_bias = bias is not None
        return linear_scaled_tf32x3(a, row_scale, weight, bias)

    @staticmethod
    def backward(ctx, gy):
        a, row_scale, weight = ctx.saved_tensors
        ga, _ = linear_bwd_tf32x3(gy, a, row_scale, weight, ctx.needs_input_grad[0], False)
        gw = library_grad_weight(gy, a, row_scale, weight) if ctx.needs_input_grad[2] else None
        gb = gy.sum(0) if (ctx.has_bias and ctx.needs_input_grad[3]) else None
        return ga, None, gw, gb


def post_linear_scaled(a: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """The caller has checked ``scaled_kernel_applies``: there is no library fallback for the compact operand."""
    if torch.is_grad_enabled() and (a.requires_grad or weight.requires_grad or (bias is not None and bias.requires_grad)):
        return _LinearScaled3xTF32.apply(a, row_scale, weight, bias)
    return linear_scaled_tf32x3(a, row_scale, weight, bias)
