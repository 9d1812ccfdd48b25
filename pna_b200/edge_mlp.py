"""The per-edge pretrans MLP of the dense layer with ``pretrans_layers = L >= 2`` (reference ``models/layers.py:200-229``)
as one libpna_sm90 call per direction: ``pna_edge_mlp_fwd`` / ``pna_edge_mlp_bwd``.

With one pretrans layer the message is affine and the dense layer gathers two node-level GEMMs.  With L >= 2 a ReLU sits
between the layers, so the message ``pretrans_t([h_i, h_j])`` has to be evaluated per edge.  The first layer still splits
into node GEMMs (``A = h W1[:, :F]^T``, ``Bm = h W1[:, F:]^T``); the kernel runs the rest of the chain in registers and
writes every message once, in CSR slot order.

Backward: the kernel stores the pre-activation gradient of every layer per slot (no atomics); the weight and bias
gradients are library GEMMs and sums (as ``linear.library_grad_weight``), and ``dA`` / ``dBm`` are the aggregation's
``sum`` over the row CSR and over its slot-transposed CSR -- fixed orders, so the whole backward is deterministic.

``edge_messages`` is the same chain for the PyG ``PNAConv`` and the DGL ``PNALayer`` (``pna_edge_msg_fwd`` /
``pna_edge_msg_bwd``): the edge-feature columns of the first layer arrive as one per-slot term ``C`` (a single GEMM over
the permuted edge features), any ``L >= 1`` is taken (``L = 1``: the message is the first layer's output, any width), and
the messages are written at the aggregation's padded tower pitch, pad columns zero, so no copy follows.

bf16 operands (the layers under bf16 autocast, DESIGN section 2): ``edge_messages`` and ``edge_mlp`` take A, Bm and C in
bfloat16 with fp32 weights and run ``pna_edge_msg_fwd_bf16`` / ``pna_edge_msg_bwd_bf16``: the messages and the stored
activations are bf16, the pre-activation gradients fp32; the result is the fp32 kernel's on the widened operands, rounded
to bf16 once.  Explicit bf16 models (bf16 weights) are not taken: the fp32-weight rule keeps them on their torch path.
"""
from __future__ import annotations

import torch

from . import _lib, capture
from .aggregate import aggregate_forward
from .csr import CSRGraph

_ID = {"log": 1.0, "lin": 1.0}

# Below this many edges a training step of the PyG / DGL layers is bound by host launch overhead, and there the torch
# message path measured faster than edge_messages (tools/edge_msg_bench.py on an H100 80GB HBM3 at 700 W: the DGL layer at
# the ZINC and MNIST shapes with 128 graphs, 6 k and 72 k edges: the order changed between runs, with kernel steps up to
# 10 % slower; from 572 k edges on, faster in every run).  The
# layers pick the torch path for such steps; forward passes without autograd always take the kernel.
FUSED_TRAINING_MIN_EDGES = 1 << 17


def _ptr(t):
    return None if t is None else t.data_ptr()


def _check(A, Bm, b1, W, bW, csr: CSRGraph, towers: int):
    L1, T, Ft, Ft2 = W.shape
    if T != towers or Ft != Ft2 or tuple(bW.shape) != (L1, T, Ft) or L1 < 1:
        raise ValueError(f"edge MLP weights must be [L-1, towers, F_t, F_t] and [L-1, towers, F_t], got {tuple(W.shape)}, "
                         f"{tuple(bW.shape)}")
    TF = T * Ft
    if A.shape != (csr.n_nodes, TF) or Bm.dim() != 2 or Bm.size(1) != TF or tuple(b1.shape) != (TF,):
        raise ValueError(f"edge MLP inputs must be A [{csr.n_nodes}, {TF}], Bm [n_src, {TF}], b1 [{TF}]")
    for t in (A, Bm, b1, W, bW):
        if t.dtype != torch.float32 or not t.is_cuda:
            raise TypeError("the edge MLP kernel takes float32 CUDA tensors")
    if Ft > _lib.EDGE_MLP_MAX_WIDTH:
        raise NotImplementedError(f"edge MLP: tower width {Ft} > {_lib.EDGE_MLP_MAX_WIDTH} is not supported by pna_edge_mlp_fwd")
    return L1 + 1, T, Ft


def edge_mlp_forward(A, Bm, b1, W, bW, csr: CSRGraph, towers: int, store_activations: bool = False):
    """Messages ``M [E, T*F_t]`` in CSR slot order (and the activations ``[L-1, E, T*F_t]`` when asked)."""
    L, T, Ft = _check(A, Bm, b1, W, bW, csr, towers)
    A, Bm, b1, W, bW = (t.contiguous() for t in (A, Bm, b1, W, bW))
    E, dev = csr.n_edges, A.device
    M = torch.empty((E, T * Ft), dtype=torch.float32, device=dev)
    act = torch.empty((L - 1, E, T * Ft), dtype=torch.float32, device=dev) if store_activations else None
    capture.pin(csr)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_edge_mlp_fwd(
            _ptr(csr.rowptr), _ptr(csr.col) if E else None, csr.n_nodes, E, _ptr(A), _ptr(Bm), _ptr(b1), _ptr(W), _ptr(bW),
            L, T, Ft, _ptr(M), _ptr(act), torch.cuda.current_stream(dev).cuda_stream))
    return M, act


def edge_mlp_backward(grad_M, act, W, n_layers: int, towers: int, width: int):
    """``[L-1, E, T*F_t]``: the per-slot pre-activation gradients G_1 .. G_(L-1) (G_L is ``grad_M``)."""
    grad_M, W = grad_M.contiguous().float(), W.contiguous()
    E, dev = grad_M.size(0), grad_M.device
    G = torch.empty((n_layers - 1, E, towers * width), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().pna_edge_mlp_bwd(_ptr(grad_M), _ptr(act), _ptr(W), E, n_layers, towers, width, _ptr(G),
                                               torch.cuda.current_stream(dev).cuda_stream))
    return G


class _EdgeMLP(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A, Bm, b1, W, bW, csr, towers):
        M, act = edge_mlp_forward(A, Bm, b1, W, bW, csr, towers, store_activations=True)
        ctx.save_for_backward(W, act)
        ctx.meta = (csr, towers, Bm.size(0))
        return M

    @staticmethod
    def backward(ctx, grad_M):
        W, act = ctx.saved_tensors
        csr, T, n_src = ctx.meta
        L, Ft = W.size(0) + 1, W.size(2)
        E = grad_M.size(0)
        G = edge_mlp_backward(grad_M, act, W, L, T, Ft)
        grads = [G[k] for k in range(L - 1)] + [grad_M.float()]      # G_1 .. G_L
        per_tower = lambda x: x.reshape(E, T, Ft)
        # layer k = 2..L: dW_k[t] = G_k[:, t]^T z_(k-1)[:, t],  db_k[t] = sum over slots of G_k[:, t]
        dW = torch.stack([torch.bmm(per_tower(grads[k - 1]).permute(1, 2, 0), per_tower(act[k - 2]).permute(1, 0, 2))
                          for k in range(2, L + 1)])
        dbW = torch.stack([per_tower(grads[k - 1]).sum(0) for k in range(2, L + 1)])
        G1 = grads[0]
        dA, dBm, db1 = _first_layer_grads(ctx, G1, csr, n_src)
        return dA, dBm, db1, dW, dbW, None, None


def _first_layer_grads(ctx, G1, csr: CSRGraph, n_src: int):
    """dA, dBm, db1 from G_1 [E, T*F_t]: sums over the slots of every row and over the out-edges of every source."""
    dA = dBm = None
    if ctx.needs_input_grad[0]:     # sum of G_1 over the slots of every row (slot order)
        dA = aggregate_forward(G1, csr, ["sum"], ["identity"], _ID, messages_in_csr_order=True)
    if ctx.needs_input_grad[1]:     # sum of G_1 over the out-edges of every source (ascending slot ids)
        dBm = aggregate_forward(G1, csr.slot_transposed(n_src), ["sum"], ["identity"], _ID)
    return dA, dBm, G1.sum(0)


def edge_mlp(A, Bm, b1, W, bW, csr: CSRGraph, towers: int) -> torch.Tensor:
    """Differentiable per-edge MLP messages ``[E, T*F_t]`` in slot order of ``csr``:
    ``M[s, t] = W_L[t] relu(... relu(A[i, t] + Bm[col[s], t] + b1[t]) ...) + b_L[t]`` (see include/pna_b200.h).
    bf16 A / Bm with fp32 weights (bf16 autocast) take ``edge_messages`` without edge term at pitch F_t: the same
    arithmetic (DESIGN section 2), with bf16 storage."""
    if A.dtype == torch.bfloat16 and W.dtype == torch.float32:
        return edge_messages(A, Bm, b1, W, bW, csr, towers)
    if torch.is_grad_enabled() and any(t.requires_grad for t in (A, Bm, b1, W, bW)):
        return _EdgeMLP.apply(A, Bm, b1, W, bW, csr, towers)
    return edge_mlp_forward(A, Bm, b1, W, bW, csr, towers)[0]


def _check_messages(A, Bm, b1, W, bW, csr: CSRGraph, towers: int, edge_term, pitch):
    """(L, T, F_t, P) of an ``edge_messages`` call; W / bW may be empty ([0, ...] or numel 0) when L = 1."""
    T = towers
    if T < 1 or A.dim() != 2 or A.size(1) % T:
        raise ValueError(f"edge messages: A must be [{csr.n_nodes}, towers * F_t] with towers = {T}")
    Ft = A.size(1) // T
    L = 1 if W.numel() == 0 else W.size(0) + 1
    if L > 1 and (tuple(W.shape) != (L - 1, T, Ft, Ft) or tuple(bW.shape) != (L - 1, T, Ft)):
        raise ValueError(f"edge MLP weights must be [L-1, {T}, {Ft}, {Ft}] and [L-1, {T}, {Ft}], got {tuple(W.shape)}, "
                         f"{tuple(bW.shape)}")
    TF = T * Ft
    if A.size(0) != csr.n_nodes or Bm.dim() != 2 or Bm.size(1) != TF or tuple(b1.shape) != (TF,):
        raise ValueError(f"edge messages: inputs must be A [{csr.n_nodes}, {TF}], Bm [n_src, {TF}], b1 [{TF}]")
    if edge_term is not None and tuple(edge_term.shape) != (csr.n_edges, TF):
        raise ValueError(f"edge messages: edge_term must be [{csr.n_edges}, {TF}] (slot order), got {tuple(edge_term.shape)}")
    P = Ft if pitch is None else int(pitch)
    if P < Ft:
        raise ValueError(f"edge messages: pitch {P} < tower width {Ft}")
    for t in (A, Bm, b1, edge_term) + ((W, bW) if L > 1 else ()):
        if t is not None and not t.is_cuda:
            raise TypeError("the edge message kernel takes CUDA tensors")
    if A.dtype not in _KERNEL or any(t is not None and t.dtype != A.dtype for t in (Bm, edge_term)):
        raise TypeError("the edge message kernel takes A, Bm and edge_term in one dtype, float32 or bfloat16")
    if any(t.dtype != torch.float32 for t in (b1,) + ((W, bW) if L > 1 else ())):
        raise TypeError("the edge message kernel takes float32 biases and weights")
    if L > 1 and Ft > _lib.EDGE_MLP_MAX_WIDTH:
        raise NotImplementedError(f"edge messages: tower width {Ft} > {_lib.EDGE_MLP_MAX_WIDTH} with {L} layers is not "
                                  "supported by pna_edge_msg_fwd")
    return L, T, Ft, P


# the entry points per storage dtype of A / Bm / C, the messages and the activations
_KERNEL = {torch.float32: ("pna_edge_msg_fwd", "pna_edge_msg_bwd"),
           torch.bfloat16: ("pna_edge_msg_fwd_bf16", "pna_edge_msg_bwd_bf16")}


def edge_messages_forward(A, Bm, b1, W, bW, csr: CSRGraph, towers: int, edge_term=None, pitch=None,
                          store_activations: bool = False):
    """Messages ``[E, T*P]`` in CSR slot order, pad columns zero (and the activations ``[L-1, E, T*F_t]`` when asked), in
    A's dtype (float32 or bfloat16)."""
    L, T, Ft, P = _check_messages(A, Bm, b1, W, bW, csr, towers, edge_term, pitch)
    A, Bm, b1 = (t.contiguous() for t in (A, Bm, b1))
    W, bW = (W.contiguous(), bW.contiguous()) if L > 1 else (None, None)
    C = None if edge_term is None else edge_term.contiguous()
    E, dev, dt = csr.n_edges, A.device, A.dtype
    M = torch.empty((E, T * P), dtype=dt, device=dev)
    act = torch.empty((L - 1, E, T * Ft), dtype=dt, device=dev) if store_activations and L > 1 else None
    capture.pin(csr)
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), _KERNEL[dt][0])(
            _ptr(csr.rowptr), _ptr(csr.col) if E else None, csr.n_nodes, E, _ptr(A), _ptr(Bm), _ptr(b1), _ptr(C), _ptr(W),
            _ptr(bW), L, T, Ft, P, _ptr(M), _ptr(act), torch.cuda.current_stream(dev).cuda_stream))
    return M, act


def edge_messages_backward(grad_M, pitch: int, act, W, n_layers: int, towers: int, width: int):
    """``[L-1, E, T*F_t]`` fp32: G_1 .. G_(L-1) from ``grad_M [E, T*pitch]`` (L >= 2), read in the activations' dtype."""
    grad_M, W = grad_M.contiguous().to(act.dtype), W.contiguous()
    E, dev = grad_M.size(0), grad_M.device
    G = torch.empty((n_layers - 1, E, towers * width), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(getattr(_lib.lib(), _KERNEL[act.dtype][1])(_ptr(grad_M), pitch, _ptr(act), _ptr(W), E, n_layers, towers,
                                                              width, _ptr(G), torch.cuda.current_stream(dev).cuda_stream))
    return G


class _EdgeMessages(torch.autograd.Function):
    @staticmethod
    def forward(ctx, A, Bm, b1, W, bW, edge_term, csr, towers, pitch):
        M, act = edge_messages_forward(A, Bm, b1, W, bW, csr, towers, edge_term, pitch, store_activations=True)
        ctx.save_for_backward(W, act)
        ctx.meta = (csr, towers, Bm.size(0), A.size(1) // towers, M.size(1) // towers)
        ctx.dtypes = (A.dtype, Bm.dtype, None if edge_term is None else edge_term.dtype)
        return M

    @staticmethod
    def backward(ctx, grad_M):
        W, act = ctx.saved_tensors
        csr, T, n_src, Ft, P = ctx.meta
        E = grad_M.size(0)
        L = 1 if act is None else W.size(0) + 1
        GL = grad_M.float().reshape(E, T, P)[:, :, :Ft]            # G_L: the unpadded columns of grad_M
        if L == 1:
            grads = [GL.reshape(E, T * Ft)]
        else:
            grads = list(edge_messages_backward(grad_M, P, act, W, L, T, Ft)) + [GL]
        dW = dbW = None
        if L > 1:
            # dW_k[t] = G_k[:, t]^T z_(k-1)[:, t] as one GEMM per tower over all E slots, db_k[t] = sum over slots of
            # G_k[:, t].  At E = 1.2 M a batched product over the towers instead took the PyG training step of
            # tools/edge_msg_bench.py to 65 ms, against 27 ms (two runs, H100 80GB HBM3, 700 W)
            cols = lambda x, t: x.reshape(E, T, Ft)[:, t]
            # (bf16 activations are widened one tower slice at a time: the weight gradients are fp32 GEMMs)
            dW = torch.stack([torch.stack([cols(grads[k - 1], t).t() @ cols(act[k - 2], t).float() for t in range(T)])
                              for k in range(2, L + 1)])
            dbW = torch.stack([grads[k - 1].reshape(E, T, Ft).sum(0) for k in range(2, L + 1)])
        dA, dBm, db1 = _first_layer_grads(ctx, grads[0], csr, n_src)
        dC = grads[0] if ctx.needs_input_grad[5] else None
        dt_a, dt_b, dt_c = ctx.dtypes        # each input's gradient in its own dtype (fp32 sums, rounded once)
        dA, dBm, dC = (None if g is None else g.to(d) for g, d in ((dA, dt_a), (dBm, dt_b), (dC, dt_c)))
        return dA, dBm, db1, dW, dbW, dC, None, None, None


def fused_step_pays(n_edges: int) -> bool:
    """Whether a layer call on ``n_edges`` edges should take edge_messages: always without autograd, with it from
    ``FUSED_TRAINING_MIN_EDGES`` edges on."""
    return not torch.is_grad_enabled() or n_edges >= FUSED_TRAINING_MIN_EDGES


def edge_messages(A, Bm, b1, W, bW, csr: CSRGraph, towers: int, edge_term=None, pitch=None) -> torch.Tensor:
    """Differentiable per-edge messages ``[E, T*P]`` in slot order of ``csr`` (P = ``pitch``, default F_t; pad columns 0):
    ``M[s, t] = W_L[t] relu(... relu(A[i, t] + Bm[col[s], t] + b1[t] + C[s, t]) ...) + b_L[t]``, or the first layer's
    output ``A[i, t] + Bm[col[s], t] + b1[t] + C[s, t]`` when ``W`` / ``bW`` are empty (L = 1).  ``edge_term`` C
    [E, T*F_t] is in slot order; its gradient is G_1 (see include/pna_b200.h)."""
    ins = (A, Bm, b1, W, bW) + (() if edge_term is None else (edge_term,))
    if torch.is_grad_enabled() and any(t.requires_grad for t in ins):
        return _EdgeMessages.apply(A, Bm, b1, W, bW, edge_term, csr, towers, pitch)
    return edge_messages_forward(A, Bm, b1, W, bW, csr, towers, edge_term, pitch)[0]
