"""Set2Set graph readout and ``S2SReadout`` (reference ``models/layers.py`` :53-98 and :271-289) on ``pna_set2set_fwd`` /
``pna_set2set_bwd``.

The reference runs ``T = steps or N`` steps of an LSTM cell, a batched matmul, a softmax and a weighted sum, each step a
handful of dependent launches.  Here one CUDA launch runs every step of every graph (one CTA per graph) and one launch
runs the back-propagation through time; the LSTM weight gradients are library fp32 GEMMs over the ``T * B`` rows of the
gate gradients the backward writes (as ``linear.library_grad_weight``).  ``Set2Set`` keeps a real ``nn.LSTM`` named
``lstm``, so parameter names, initialisation and reference ``state_dict``s are the reference's.

fp32 only.  Inside ``torch.autocast("cuda")`` an fp16 / bf16 ``x`` is upcast to fp32 at the kernel boundary and the output
is fp32 (the reference would run its LSTM in the autocast dtype; DESIGN section 9).  There is no CPU path.
"""
from __future__ import annotations

import ctypes as C

import torch
import torch.nn as nn

from . import _lib
from .nn_blocks import MLP

__all__ = ["Set2Set", "S2SReadout", "set2set", "saved_floats"]


def saved_floats(n_graphs: int, n_nodes: int, n_feat: int, steps: int) -> int:
    """Size in floats of the buffer the forward saves for the backward (``pna_set2set_saved_floats``)."""
    n = C.c_int64(0)
    _lib.check(_lib.lib().pna_set2set_saved_floats(n_graphs, n_nodes, n_feat, steps, C.byref(n)))
    return n.value


def _check_limits(n_nodes: int, n_feat: int) -> None:
    if n_feat > _lib.SET2SET_MAX_FEAT or n_nodes * n_feat > _lib.SET2SET_MAX_ELEMS:
        raise NotImplementedError(f"Set2Set kernel takes n_feat <= {_lib.SET2SET_MAX_FEAT} and n_nodes * n_feat <= "
                                  f"{_lib.SET2SET_MAX_ELEMS}, got n_nodes={n_nodes}, n_feat={n_feat}")


class _Set2SetFn(torch.autograd.Function):
    """Saves the forward's per-step records (q*, c, gate activations, attention) only when a gradient is needed."""

    @staticmethod
    def forward(ctx, x, steps, need_grad, w_ih, w_hh, b_ih, b_hh):
        B, N, D = x.shape
        out = torch.empty(B, 2 * D, device=x.device, dtype=torch.float32)
        saved = torch.empty(saved_floats(B, N, D, steps), device=x.device, dtype=torch.float32) if need_grad else None
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().pna_set2set_fwd(x.data_ptr(), B, N, D, steps, w_ih.data_ptr(), w_hh.data_ptr(), b_ih.data_ptr(),
                                                  b_hh.data_ptr(), out.data_ptr(), None if saved is None else saved.data_ptr(),
                                                  torch.cuda.current_stream(x.device).cuda_stream))
        if need_grad:
            ctx.save_for_backward(x, w_ih, w_hh, saved)
            ctx.steps = steps
        return out

    @staticmethod
    def backward(ctx, grad_out):
        want_x, _, _, want_ih, want_hh, want_bih, want_bhh = ctx.needs_input_grad
        if not (want_x or want_ih or want_hh or want_bih or want_bhh):
            return (None,) * 7
        x, w_ih, w_hh, saved = ctx.saved_tensors
        B, N, D = x.shape
        T = ctx.steps
        grad_out = grad_out.float().contiguous()
        gx = torch.empty_like(x) if want_x else None
        gates = torch.empty(T * B, 4 * D, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _lib.check(_lib.lib().pna_set2set_bwd(x.data_ptr(), B, N, D, T, w_ih.data_ptr(), w_hh.data_ptr(), saved.data_ptr(),
                                                  grad_out.data_ptr(), None if gx is None else gx.data_ptr(), gates.data_ptr(),
                                                  torch.cuda.current_stream(x.device).cuda_stream))
        # step t's LSTM input is q*_{t-1} (zero at t = 0): the GEMMs pair gate rows t >= 1 with the q* rows of step t - 1,
        # read in place from the saved records (pitch 7D + N)
        q_prev = saved.view(T * B, 7 * D + N)[:(T - 1) * B, :2 * D]
        g_next = gates[B:]
        with torch.autocast("cuda", enabled=False):
            gw_ih = g_next.t() @ q_prev if want_ih else None
            gw_hh = g_next.t() @ q_prev[:, :D] if want_hh else None
            gb = gates.sum(0) if (want_bih or want_bhh) else None
        gb_ih = gb if want_bih else None
        gb_hh = None if not want_bhh else gb.clone() if want_bih else gb      # two parameters never share one grad tensor
        return gx, None, None, gw_ih, gw_hh, gb_ih, gb_hh


def set2set(x: torch.Tensor, steps, w_ih: torch.Tensor, w_hh: torch.Tensor, b_ih: torch.Tensor, b_hh: torch.Tensor) -> torch.Tensor:
    """Set2Set of ``x [B, N, D]`` with the one-layer LSTM ``(w_ih [4D, 2D], w_hh [4D, D], b_ih [4D], b_hh [4D])`` over
    ``steps or N`` steps -> ``q* [B, 2D]`` (fp32).  Differentiable in ``x`` and the four weights."""
    if x.dim() != 3:
        raise ValueError(f"Set2Set input must be [B, N, D], got {tuple(x.shape)}")
    if not x.is_cuda:
        raise ValueError("pna_b200 Set2Set runs on CUDA tensors only (no CPU fallback)")
    if x.dtype in (torch.float16, torch.bfloat16) and torch.is_autocast_enabled("cuda"):
        x = x.float()                                   # the kernel boundary of an autocast region: fp32 in, fp32 out
    B, N, D = x.shape
    for name, t, shape in (("x", x, None), ("weight_ih", w_ih, (4 * D, 2 * D)), ("weight_hh", w_hh, (4 * D, D)),
                           ("bias_ih", b_ih, (4 * D,)), ("bias_hh", b_hh, (4 * D,))):
        if t.dtype != torch.float32:
            raise TypeError(f"Set2Set kernel is fp32 only: {name} is {t.dtype}")
        if t.device != x.device:
            raise ValueError(f"Set2Set: {name} is on {t.device}, x on {x.device}")
        if shape is not None and tuple(t.shape) != shape:
            raise ValueError(f"Set2Set: {name} has shape {tuple(t.shape)}, expected {shape}")
    T = int(steps or N)
    if B == 0 or T == 0:                                # no graph, or no node and no step: q* stays zero
        return x.new_zeros(B, 2 * D)
    if N == 0:
        raise NotImplementedError("Set2Set with explicit steps over graphs of zero nodes (an empty softmax) is not supported")
    _check_limits(N, D)
    params = (w_ih, w_hh, b_ih, b_hh)
    need_grad = torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params))
    return _Set2SetFn.apply(x.contiguous(), T, need_grad, *(p.contiguous() for p in params))


class Set2Set(nn.Module):
    """Drop-in for the reference's ``Set2Set`` (``models/layers.py`` :53-98) on ``x [B, N, D]``; see :func:`set2set`.

    ``num_layers != 1`` raises ``NotImplementedError``; ``nhid != 2 * nin`` is accepted here (as in the reference, whose
    LSTM then fails on its second step) and raises ``ValueError`` in ``forward``.  ``activation`` is ignored, as in the
    reference."""

    def __init__(self, nin, nhid=None, steps=None, num_layers=1, activation=None, device="cpu"):
        super().__init__()
        self.steps = steps
        self.nin = nin
        self.nhid = nin * 2 if nhid is None else nhid
        if self.nhid <= self.nin:
            raise ValueError("Set2Set hidden_dim should be larger than input_dim")
        if num_layers != 1:
            raise NotImplementedError("pna_b200 Set2Set supports num_layers=1 only (the reference's S2SReadout)")
        self.lstm_output_dim = self.nhid - self.nin
        self.num_layers = num_layers
        self.lstm = nn.LSTM(self.nhid, self.nin, num_layers=num_layers, batch_first=True).to(device)

    def forward(self, x):
        if self.nhid != 2 * self.nin:
            raise ValueError(f"Set2Set needs nhid == 2 * nin (the LSTM input is [q, r]), got nin={self.nin}, nhid={self.nhid}")
        if x.dim() != 3 or x.size(2) != self.nin:
            raise ValueError(f"Set2Set({self.nin}) input must be [B, N, {self.nin}], got {tuple(x.shape)}")
        L = self.lstm
        return set2set(x, self.steps, L.weight_ih_l0, L.weight_hh_l0, L.bias_ih_l0, L.bias_hh_l0)


class S2SReadout(nn.Module):
    """Drop-in for the reference's ``S2SReadout`` (``models/layers.py`` :271-289): ``Set2Set(in_size)`` then an MLP with
    batch norm between its layers.  Keys ``set2set.lstm.*`` and ``mlp.fully_connected.{k}.{linear,b_norm}.*``."""

    def __init__(self, in_size, hidden_size, out_size, fc_layers=3, device="cpu", final_activation="relu"):
        super().__init__()
        self.set2set = Set2Set(in_size, device=device)
        self.mlp = MLP(in_size=2 * in_size, hidden_size=hidden_size, out_size=out_size, layers=fc_layers, mid_activation="relu",
                       last_activation=final_activation, mid_b_norm=True, last_b_norm=False, device=device)

    def forward(self, x):
        return self.mlp(self.set2set(x))
