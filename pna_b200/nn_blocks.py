"""Dense building blocks the DGL- and dense-signature layers are assembled from.

Parameter names and forward order match reference ``models/layers.py`` (``FCLayer`` :101-197, ``MLP`` :200-234) so
reference ``state_dict``s load unchanged: ``fully_connected.{k}.linear.{weight,bias}`` (+ ``b_norm.*``).
These are plain torch.nn glue (cuBLAS linears); the hot path is the aggregation kernel, not this file.
"""
from __future__ import annotations

import torch
import torch.nn as nn

_ACTIVATIONS = {"relu": nn.ReLU, "sigmoid": nn.Sigmoid, "tanh": nn.Tanh, "elu": nn.ELU, "selu": nn.SELU, "glu": nn.GLU,
                "leakyrelu": nn.LeakyReLU, "softplus": nn.Softplus}


def make_activation(spec):
    """Name (case-insensitive, 'none' -> no activation) or callable -> module / None (layers.py:8-19)."""
    if spec is not None and callable(spec):
        return spec
    key = str(spec).lower()
    if key == "none":
        return None
    if key not in _ACTIVATIONS:
        raise AssertionError("Unhandled activation function")
    return _ACTIVATIONS[key]()


class FCLayer(nn.Module):
    """Linear -> activation -> dropout -> batch norm, Xavier-uniform weight with gain 1/in_size, zero bias."""

    def __init__(self, in_size, out_size, activation="relu", dropout=0.0, b_norm=False, bias=True, init_fn=None,
                 device="cpu"):
        super().__init__()
        self.in_size, self.out_size, self.bias = in_size, out_size, bias
        self.linear = nn.Linear(in_size, out_size, bias=bias).to(device)
        self.dropout = nn.Dropout(p=dropout) if dropout else None
        self.b_norm = nn.BatchNorm1d(out_size).to(device) if b_norm else None
        self.activation = make_activation(activation)
        self.init_fn = init_fn or nn.init.xavier_uniform_
        self.reset_parameters()

    def reset_parameters(self, init_fn=None):
        init_fn = init_fn or self.init_fn
        if init_fn is not None:
            init_fn(self.linear.weight, 1 / self.in_size)
        if self.bias:
            self.linear.bias.data.zero_()

    def forward(self, x, weight=None, row_scale=None):
        """`weight`: optional replacement for linear.weight (same parameters, zero columns inserted for padded inputs).
        `row_scale` [N, S]: x is the compact aggregate and the S scaled copies are formed inside the kernel (linear.py)."""
        if row_scale is not None:
            from .linear import post_linear_scaled
            h = post_linear_scaled(x, row_scale, self.linear.weight if weight is None else weight, self.linear.bias)
        elif x.dim() == 2:   # tensor-core path for the shapes pna_linear_fwd takes, library GEMM otherwise
            from .linear import post_linear
            h = post_linear(x, self.linear.weight if weight is None else weight, self.linear.bias)
        else:
            h = self.linear(x) if weight is None else nn.functional.linear(x, weight, self.linear.bias)
        return self.after_linear(h)

    def after_linear(self, h):
        """activation -> dropout -> batch norm on the output of this layer's Linear (computed by the caller)."""
        if self.activation is not None:
            h = self.activation(h)
        if self.dropout is not None:
            h = self.dropout(h)
        if self.b_norm is not None:
            h = self.b_norm(h.transpose(1, 2)).transpose(1, 2) if h.shape[1] != self.out_size else self.b_norm(h)
        return h

    def __repr__(self):
        return f"{self.__class__.__name__} ({self.in_size} -> {self.out_size})"


class MLP(nn.Module):
    """A stack of FCLayers: in -> hidden x (layers-1) -> out (layers.py:200-234)."""

    def __init__(self, in_size, hidden_size, out_size, layers, mid_activation="relu", last_activation="none", dropout=0.0,
                 mid_b_norm=False, last_b_norm=False, device="cpu"):
        super().__init__()
        self.in_size, self.hidden_size, self.out_size = in_size, hidden_size, out_size
        sizes = [in_size] + [hidden_size] * (max(layers, 1) - 1) + [out_size]
        self.fully_connected = nn.ModuleList()
        for k in range(len(sizes) - 1):
            last = k == len(sizes) - 2
            self.fully_connected.append(FCLayer(sizes[k], sizes[k + 1], activation=last_activation if last else mid_activation,
                                                b_norm=last_b_norm if last else mid_b_norm, device=device, dropout=dropout))

    def forward(self, x, first_weight=None, first_row_scale=None):
        for k, fc in enumerate(self.fully_connected):
            x = fc(x, first_weight, first_row_scale) if k == 0 else fc(x)
        return x

    def is_single_affine(self) -> bool:
        """True when the MLP is one Linear without activation / dropout / norm: the message is affine in its inputs."""
        fc = self.fully_connected[0]
        return len(self.fully_connected) == 1 and fc.activation is None and fc.dropout is None and fc.b_norm is None

    def is_linear_relu(self) -> bool:
        """True when every layer is a bare Linear with a ReLU between layers and none after the last: the stack the
        per-edge message kernels (edge_mlp.py) evaluate."""
        fcs = self.fully_connected
        return not any(fc.dropout is not None or fc.b_norm is not None for fc in fcs) and \
            all(isinstance(fc.activation, nn.ReLU) for fc in fcs[:-1]) and fcs[-1].activation is None

    def __repr__(self):
        return f"{self.__class__.__name__} ({self.in_size} -> {self.out_size})"
