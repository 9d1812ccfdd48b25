"""First dense linear of the post-aggregation MLP on the H100 tensor cores (``pna_linear_fwd``, 3xTF32 wgmma).

``post_linear(a, weight, bias)`` is ``torch.nn.functional.linear`` for the shapes the kernel takes
(fp32, in_features % 32 == 0, out_features in {64, 128, 256}) and falls back to the library GEMM for every other shape --
the kernel is an accelerator for one GEMM shape family, not a requirement of the path.

``post_linear_scaled(a, row_scale, weight, bias)`` is the same linear fed by the COMPACT aggregate (SURVEY 8(f)-2):
``a`` is the ``[N, A*F]`` result of the identity scaler alone and the S scaled copies the reference concatenates
(pna.py:247-249) are regenerated in registers by the kernel's loaders -- ``linear(cat_s(row_scale[:, s:s+1] * a), W, b)``
without the ``[N, S*A*F]`` tensor ever being written or read.

``post_linear_towers_scaled(a, row_scale, weight, bias)`` is the compact path of the tower layers (PNAConv, the DGL
PNALayer): ``a`` holds per tower ``[self | A aggregates]`` and every tower's first post Linear runs in one kernel on that
tower's columns, the scaled copies formed in registers (``pna_linear_towers_scaled_fwd`` / ``pna_linear_towers_bwd_data``).

Backward: the input gradient runs on the tensor cores (``pna_linear_bwd_data``, same accuracy, no atomics; the compact one
never forms the scaled copies).  The weight gradient stays a library fp32 GEMM (``library_grad_weight``): at config 2 on
H100 cuBLAS is faster than the tensor-core ``pna_linear_bwd_weight`` (DESIGN section 5), which ``linear_bwd_tf32x3``
still exposes.

Every wrapper of a C entry point checks its operands' dtypes before it allocates or launches anything (``_fp32``): the C
side takes ``const float*`` and cannot tell a bf16 buffer from an fp32 one.  The one bf16 operand taken is the compact
tower aggregate (``pna_linear_towers_scaled_fwd_bf16``, the tower layers under bf16 autocast): its output, the data
gradient and the weight gradient stay fp32, and the data gradient is returned in bf16, the aggregate's dtype.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _lib, aggregate

_OUT_OK = (64, 128, 256)


def kernel_applies(a: torch.Tensor, weight: torch.Tensor) -> bool:
    if os.environ.get("PNA_B200_TENSOR_LINEAR", "1") == "0":       # opt out: keep the library fp32 GEMM
        return False
    return (a.is_cuda and a.dtype == torch.float32 and weight.dtype == torch.float32 and a.dim() == 2 and a.size(0) > 0
            and a.size(1) % 32 == 0 and weight.size(0) in _OUT_OK and a.stride(1) == 1 and a.stride(0) % 4 == 0
            and a.data_ptr() % 16 == 0)


def _fp32(who: str, **operands) -> None:
    """TypeError unless every given operand is float32 (None: absent)."""
    for name, t in operands.items():
        if t is not None and t.dtype != torch.float32:
            raise TypeError(f"{who}: {name} is {t.dtype}; the kernel takes float32")


def linear_tf32x3(a: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor]) -> torch.Tensor:
    """y = a @ weight.T + bias through the C ABI (no autograd)."""
    _fp32("linear_tf32x3", a=a, weight=weight, bias=bias)
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
    _fp32("linear_bwd_tf32x3", gy=gy, a=a, row_scale=row_scale, weight=weight)
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
    _fp32("linear_scaled_tf32x3", a=a, row_scale=row_scale, weight=weight, bias=bias)
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


# ---- tower layers (PNAConv, the DGL PNALayer): per tower a = [self | A aggregates], the scaled copies inside the kernel ----
TOWERS_MAX = 8          # pna_linear_towers_*: n_towers <= 8, n_out <= 64 per tower, n_towers * n_out <= 256, n_feat % 4 == 0
TOWER_OUT_MAX = 64


def towers_path_ok(x: torch.Tensor, n_towers: int, n_feat: int, n_out: int, n_scalers: int) -> bool:
    """Shape-level decision the tower layers take BEFORE aggregating: would a fresh fp32 [N, T * (1 + A) * n_feat] compact
    aggregate on x's device, with [T, n_out, (1 + S * A) * n_feat] first post Linears, go through
    pna_linear_towers_scaled_fwd?  (The layers check the weights' dtype themselves.)  Inside autocast the aggregate has the
    boundary dtype whatever x's (fp32, or bf16 for pna_linear_towers_scaled_fwd_bf16), so x's dtype is not asked."""
    dtype_ok = aggregate.boundary_dtype() is not None or x.dtype == torch.float32
    return (n_scalers > 1 and x.is_cuda and dtype_ok and x.size(0) > 0 and 1 <= n_towers <= TOWERS_MAX
            and 1 <= n_out <= TOWER_OUT_MAX and n_towers * n_out <= 256 and n_feat % 4 == 0
            and os.environ.get("PNA_B200_TENSOR_LINEAR", "1") != "0" and os.environ.get("PNA_B200_COMPACT_POST", "1") != "0")


# Training steps on graphs of at least this many rows take the compact tower path.  Measured on an H100 80GB HBM3 at
# 700 W (tools/tower_post_bench.py): the step is faster from the arxiv shape up (169 k rows: 10.4 vs 13.8 ms, ZINC
# 12 000 graphs, 278 k rows: 49.6 vs 53.4 ms) and slower on 128-graph batches (3 k / 9 k rows: +0.5 / +0.8 ms of
# launches: one weight-gradient GEMM per tower and scaler); sizes in between were not measured.  A forward without
# autograd keeps the materialised path: the kernel's forward is slower than the library GEMM it replaces (3.8 vs 3.0 ms).
TOWERS_COMPACT_MIN_ROWS = 100_000


def towers_compact_pays(n_rows: int, training: bool) -> bool:
    return training and n_rows >= TOWERS_COMPACT_MIN_ROWS


def _tower_dims(a: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor):
    """(T, O_t, Fp, A) from a [N, T * (1 + A) * Fp], row_scale [N, S], weight [T, O_t, (1 + S * A) * Fp]."""
    t, o, kw = weight.shape
    s = row_scale.size(1)
    per = a.size(1) // t                          # (1 + A) * Fp
    af = (kw - per) // (s - 1) if s > 1 else -1   # A * Fp
    fp = per - af
    if (s < 2 or a.size(1) != t * per or af <= 0 or fp <= 0 or af % fp or kw != fp + s * af or row_scale.size(0) != a.size(0)
            or row_scale.dtype != torch.float32 or not row_scale.is_contiguous()):
        raise ValueError("need a [N, T*(1+A)*Fp], row_scale a contiguous fp32 [N, S] with S > 1, weight [T, O_t, (1+S*A)*Fp]")
    return t, o, fp, af // fp


def linear_towers_scaled_tf32x3(a: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor,
                                bias: Optional[torch.Tensor]) -> torch.Tensor:
    """y[:, t*O_t:(t+1)*O_t] = [self_t | cat_s(row_scale[:, s, None] * agg_t)] @ weight[t].T + bias[t] through the C ABI
    (no autograd); a's tower block t is [self_t | agg_t].  a may be bf16 (pna_linear_towers_scaled_fwd_bf16: y is then
    what the fp32 call gives on a.float(), bit for bit); y is fp32 either way."""
    _fp32("linear_towers_scaled_tf32x3", a=None if a.dtype == torch.bfloat16 else a, row_scale=row_scale, weight=weight,
          bias=bias)
    t, o, fp, n_aggr = _tower_dims(a, row_scale, weight)
    a = a.contiguous()
    n = a.size(0)
    dev = a.device
    w = weight.detach().contiguous()
    b = None if bias is None else bias.detach().contiguous()
    y = torch.empty((n, t * o), dtype=torch.float32, device=dev)
    entry = "pna_linear_towers_scaled_fwd_bf16" if a.dtype == torch.bfloat16 else "pna_linear_towers_scaled_fwd"
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), entry)(a.data_ptr(), a.stride(0), row_scale.data_ptr(), row_scale.size(1), w.data_ptr(),
                                              None if b is None else b.data_ptr(), y.data_ptr(), y.stride(0), n, t, fp, n_aggr, o,
                                              torch.cuda.current_stream(dev).cuda_stream))
    return y


def linear_towers_bwd_data(gy: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor, a_shape) -> torch.Tensor:
    """grad a of ``linear_towers_scaled_tf32x3`` (no autograd): self columns sum_o gy W_self, aggregate columns
    sum_s fl(c_s gy) W_s, the scaled copies of gy formed in the kernel's loaders.  fp32 result."""
    _fp32("linear_towers_bwd_data", gy=gy, row_scale=row_scale, weight=weight)
    t, o, fp, n_aggr = _tower_dims(torch.empty(a_shape, device="meta"), row_scale, weight)
    gy = gy.contiguous()
    n = a_shape[0]
    dev = gy.device
    w = weight.detach().contiguous()
    ga = torch.empty(a_shape, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_linear_towers_bwd_data(gy.data_ptr(), gy.stride(0), row_scale.data_ptr(), row_scale.size(1), w.data_ptr(),
                                                         ga.data_ptr(), ga.stride(0), n, t, fp, n_aggr, o,
                                                         torch.cuda.current_stream(dev).cuda_stream))
    return ga


def library_grad_weight_towers(gy: torch.Tensor, a: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """grad weight of ``linear_towers_scaled_tf32x3``: library fp32 GEMMs, one per tower for the self block and one per
    tower and scaler for the aggregates, each ``fl(c_s * agg_t)`` a temporary of one tower's aggregate block.  A bf16 a is
    widened one tower block at a time, never as a whole."""
    t, o, fp, n_aggr = _tower_dims(a, row_scale, weight)
    af, per = n_aggr * fp, (1 + n_aggr) * fp
    gw = torch.empty_like(weight)
    for k in range(t):
        gy_t, a_t = gy[:, k * o:(k + 1) * o], a[:, k * per:(k + 1) * per].float()
        torch.mm(gy_t.t(), a_t[:, :fp], out=gw[k, :, :fp])
        for s in range(row_scale.size(1)):
            torch.mm(gy_t.t(), a_t[:, fp:] * row_scale[:, s:s + 1], out=gw[k, :, fp + s * af:fp + (s + 1) * af])
    return gw


class _LinearTowersScaled3xTF32(torch.autograd.Function):
    """Saves the compact aggregate (bf16 under bf16 autocast: half the bytes), not the scaled copies.  The scale factors are
    constants of the graph.  The data gradient is returned in a's dtype."""

    @staticmethod
    def forward(ctx, a, row_scale, weight, bias):
        ctx.save_for_backward(a, row_scale, weight)
        ctx.has_bias = bias is not None
        return linear_towers_scaled_tf32x3(a, row_scale, weight, bias)

    @staticmethod
    def backward(ctx, gy):
        a, row_scale, weight = ctx.saved_tensors
        ga = linear_towers_bwd_data(gy, row_scale, weight, a.shape).to(a.dtype) if ctx.needs_input_grad[0] else None
        gw = library_grad_weight_towers(gy, a, row_scale, weight) if ctx.needs_input_grad[2] else None
        gb = gy.sum(0).view(weight.size(0), weight.size(1)) if (ctx.has_bias and ctx.needs_input_grad[3]) else None
        return ga, None, gw, gb


def post_linear_towers_scaled(a: torch.Tensor, row_scale: torch.Tensor, weight: torch.Tensor,
                              bias: Optional[torch.Tensor]) -> torch.Tensor:
    """First post Linear of every tower on the compact tower aggregate: a [N, T*(1+A)*Fp] (per tower [self | A aggregates],
    identity scaler only), row_scale [N, S], weight [T, O_t, (1+S*A)*Fp] (the reference's column layout with zero columns
    at the pad positions), bias [T, O_t] -> [N, T*O_t] = torch.cat over the towers.  The caller has checked
    ``towers_path_ok``: there is no library fallback for the compact operand."""
    if torch.is_grad_enabled() and (a.requires_grad or weight.requires_grad or (bias is not None and bias.requires_grad)):
        return _LinearTowersScaled3xTF32.apply(a, row_scale, weight, bias)
    return linear_towers_scaled_tf32x3(a, row_scale, weight, bias)
