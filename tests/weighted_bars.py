"""Accuracy bars of softmax / softmin / normalised_mean (DESIGN.md section 2), shared by the CPU and GPU tests.

y is measured against a float64 evaluation of the same formula on the same fp32 (or bf16-converted) messages, u = 2^-24.

softmax / softmin (n = sigma m, M = max n, p_s = exp(n_s - M) / Z, y' = sum p_s n_s):
  * u_s = fl(n_s - M) is off by at most u |n_s - M|, and expf by 2 ulp (4 u), so e_s carries a relative error of at most
    u (|n_s - M| + 4); moving e_s by a relative eps_s moves y' by sum p_s eps_s (n_s - y');
  * the products e_s n_s, the two fp32 sums of d positive / mixed terms and the division add about
    (2 + 2 sqrt(d)) u sum p_s |n_s| (the sums' rounding errors grow like sqrt(d), 2 sigma);
  bar = 2 u [ sum p_s |n_s - y'| (|n_s - M| + 4) + (2 + 2 sqrt(d)) sum p_s |n_s| ] + 2 ulp(y)   (safety factor 2).
normalised_mean: r_i, r_j (correctly rounded), their product and m_s w_s are one rounding each, then the fp32 sum:
  bar = (4 + 2 sqrt(d)) u sum |m_s| w_s + ulp(y).
Gradients are bounded term by term (see the functions), with a safety factor.
"""
import torch

import weighted_oracle as WO

U = 2.0 ** -24


def _softmax_parts(msg, dst, n, sigma):
    m = msg.double()
    F = m.size(1)
    nn_ = sigma * m
    deg = WO.in_degree(dst, n)
    M = torch.full((n, F), -float("inf"), dtype=torch.float64).index_reduce(0, dst, nn_, "amax")
    e = torch.exp(nn_ - M[dst])
    Z = torch.zeros(n, F, dtype=torch.float64).index_add(0, dst, e)
    Zs = torch.where(deg[:, None] > 0, Z, torch.ones_like(Z))
    p = e / Zs[dst]
    yp = torch.zeros(n, F, dtype=torch.float64).index_add(0, dst, p * nn_)
    return nn_, deg, M, p, yp


def softmax_bar(msg, dst, n, sigma):
    """(y64 [n, F], tol [n, F]) of softmax (sigma = 1) or softmin (sigma = -1) of per-edge messages msg [E, F]."""
    nn_, deg, M, p, yp = _softmax_parts(msg, dst, n, sigma)
    spread = torch.zeros_like(yp).index_add(0, dst, p * (nn_ - yp[dst]).abs() * ((nn_ - M[dst]).abs() + 4))
    size = torch.zeros_like(yp).index_add(0, dst, p * nn_.abs())
    c = (2 + 2 * deg.clamp(min=1).sqrt()).unsqueeze(1)
    tol = 2 * U * (spread + c * size) + 2 * 2.0 ** -23 * yp.abs()
    live = deg[:, None] > 0
    return torch.where(live, sigma * yp, torch.zeros_like(yp)), torch.where(live, tol, torch.zeros_like(tol))


def nmean_bar(msg, dst, wsrc, n):
    """(y64, tol) of normalised_mean; wsrc: the source node of every edge."""
    m = msg.double()
    w = WO.weights(dst, wsrc, n)[:, None]
    deg = WO.in_degree(dst, n)
    y = torch.zeros(n, m.size(1), dtype=torch.float64).index_add(0, dst, m * w)
    size = torch.zeros_like(y).index_add(0, dst, m.abs() * w)
    c = (4 + 2 * deg.clamp(min=1).sqrt()).unsqueeze(1)
    return y, c * U * size + 2.0 ** -23 * y.abs()


def bar(name, msg, dst, n, wsrc=None):
    if name == "normalised_mean":
        return nmean_bar(msg, dst, wsrc, n)
    return softmax_bar(msg, dst, n, -1.0 if name == "softmin" else 1.0)


def grad_bar(name, msg, dst, n, G, Gabs=None, wsrc=None, scale=4.0):
    """Float64 gradient of sum G * y (G [n, F]: the upstream gradient of y, Gabs: the sum of |scale * grad_out| it was
    formed from, default |G|) w.r.t. every message [E, F], and its bar, per slot j of row i:
      softmax / softmin:  |G| p_j [ |1 + n_j - y'| (u (|n_j - M| + 4) + eps_Z + 4 u) + u (|n_j| + |y'|) + bar(y') ]
                          + 8 u Gabs p_j |1 + n_j - y'|,   eps_Z = u sum p_s (|n_s - M| + 4) + 2 sqrt(d) u
                          (the errors of e_j, of Z, of the three roundings of the slot term, of n_j - y', and of G);
      normalised_mean:    (4 |G| + 8 Gabs) u w_j;
    times a safety factor `scale`."""
    G = G.double()
    Gabs = G.abs() if Gabs is None else Gabs.double()
    m = msg.double().clone().requires_grad_(True)
    y = WO.weighted_rows(m, dst, n, name, wsrc)
    g64, = torch.autograd.grad((y * G).sum(), m)
    if name == "normalised_mean":
        w = WO.weights(dst, wsrc, n)[:, None]
        return g64, scale * (4 * G.abs() + 8 * Gabs)[dst] * U * w
    sigma = -1.0 if name == "softmin" else 1.0
    nn_, deg, M, p, yp = _softmax_parts(msg, dst, n, sigma)
    _, ytol = softmax_bar(msg, dst, n, sigma)
    epsZ = U * torch.zeros_like(yp).index_add(0, dst, p * ((nn_ - M[dst]).abs() + 4)) + 2 * deg.clamp(min=1).sqrt()[:, None] * U
    lin = (1 + nn_ - yp[dst]).abs()
    t = G.abs()[dst] * p * (lin * (U * ((nn_ - M[dst]).abs() + 4) + epsZ[dst] + 4 * U) + U * (nn_.abs() + yp.abs()[dst]) + ytol[dst])
    t = t + 8 * U * Gabs[dst] * p * lin
    return g64, scale * t
