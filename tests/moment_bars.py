"""Accuracy bars of the moment aggregators (DESIGN.md section 2), shared by the CPU and GPU moment tests.

r_k = sign(M_k) (|M_k| + 1e-5)^(1/k) is measured against a float64 evaluation of the same formula on the same fp32 (or
bf16-converted) messages.  The fp32 error of M_k is bounded by  c * u * cond_M  with u = 2^-24 and
    cond_M = (1/d) sum |delta_s|^k + k (|mu| + max |m_s|) (1/d) sum |delta_s|^(k-1)
(the first term: the k roundings of every power, the sum and the division; the second: the error of mu and of delta = m - mu,
both ~ (|mu| + |m|) u, carried through d delta^k / d delta = k delta^(k-1)).  The root multiplies it by
rho_k = (1/k) (|M_k| + 1e-5)^(1/k - 1), then powf and the final rounding add a few ulp of r_k.  The constant
    c = k + 4 + 2 sqrt(d)
covers the k + 2 roundings per slot, the mean and the division, and a fp32 sum of d terms whose rounding errors grow like
sqrt(d) (2 sigma); the chunked sums of split rows grow slower than that.  Where M_k is within that error of 0, sign(M_k) may
come out either way: r_k may then be off by 2 (|M_k| + err + 1e-5)^(1/k), and rho_k may be at its largest.  Gradients get
the same treatment, term by term.
"""
import torch

U = 2.0 ** -24
EPS = 1e-5


def _rows(msg64, dst, n):
    deg = torch.zeros(n, dtype=torch.float64).index_add_(0, dst, torch.ones(dst.numel(), dtype=torch.float64))
    cnt = deg.clamp(min=1).unsqueeze(1)
    mu = torch.zeros(n, msg64.size(1), dtype=torch.float64).index_add(0, dst, msg64) / cnt
    return deg, cnt, mu


def moment_bar(msg, dst, n, k, ulps=4.0):
    """(r64 [n, F], tol [n, F]): float64 r_k of per-edge messages msg [E, F] by destination, and the bar of the fp32 result."""
    m = msg.double()
    deg, cnt, mu = _rows(m, dst, n)
    delta = m - mu[dst]
    M = torch.zeros_like(mu).index_add(0, dst, delta ** k) / cnt
    r = torch.sign(M) * (M.abs() + EPS) ** (1.0 / k)
    r = torch.where(deg.unsqueeze(1) > 0, r, torch.zeros_like(r))
    absk = torch.zeros_like(mu).index_add(0, dst, delta.abs() ** k) / cnt
    absk1 = torch.zeros_like(mu).index_add(0, dst, delta.abs() ** (k - 1)) / cnt
    mmax = torch.zeros_like(mu).index_reduce(0, dst, m.abs(), "amax", include_self=True)
    cond = absk + k * (mu.abs() + mmax) * absk1
    rho = (1.0 / k) * (M.abs() + EPS) ** (1.0 / k - 1.0)
    c = k + 4 + 2 * deg.clamp(min=1).sqrt().unsqueeze(1)
    errM = c * cond * U
    # sign(M) is discontinuous at 0: where M_k is within its rounding error of 0 (e.g. an odd moment of a symmetric
    # neighbourhood), fp32 may land on either side, and r_k on +-(|M| + 1e-5)^(1/k)
    jump = torch.where(M.abs() <= errM, 2 * (M.abs() + errM + EPS) ** (1.0 / k), torch.zeros_like(M))
    tol = c * rho * cond * U + ulps * r.abs() * 2.0 ** -23 + jump
    return r, tol


def moment_grad_bar(msg, dst, n, ks, G, scale=8.0):
    """Float64 gradient of sum_k G[k] * r_k (G: {k: [n, F] upstream gradient of r_k}) w.r.t. every message [E, F], and its
    bar: per slot and k,  c * u * |G k / d| rho_k (|delta_j|^(k-1) + (1/d) sum |delta|^(k-1)
    + (k-1) (|mu| + max |m|) (|delta_j|^(k-2) + (1/d) sum |delta|^(k-2)))  plus the error of rho_k carried from M_k,
    |G k / d| |d rho / dM| err(M_k) (|delta_j|^(k-1) + |C_(k-1)|), times a safety factor `scale`."""
    m = msg.double().clone().requires_grad_(True)
    deg, cnt, mu = _rows(m.detach(), dst, n)
    # autograd of the float64 formula
    deg_, cnt_, mu_ = _rows(m, dst, n)
    total = 0
    for k in ks:
        Mk = torch.zeros_like(mu_).index_add(0, dst, (m - mu_[dst]) ** k) / cnt_
        rk = torch.sign(Mk) * (Mk.abs() + EPS) ** (1.0 / k)
        total = total + (rk * G[k].double()).sum()
    g64, = torch.autograd.grad(total, m)
    delta = m.detach() - mu[dst]
    tol = torch.zeros_like(g64)
    for k in ks:
        M = torch.zeros_like(mu).index_add(0, dst, delta ** k) / cnt
        C = torch.zeros_like(mu).index_add(0, dst, delta ** (k - 1)) / cnt
        absk = torch.zeros_like(mu).index_add(0, dst, delta.abs() ** k) / cnt
        absk1 = torch.zeros_like(mu).index_add(0, dst, delta.abs() ** (k - 1)) / cnt
        mmax = torch.zeros_like(mu).index_reduce(0, dst, m.detach().abs(), "amax", include_self=True)
        c = k + 4 + 2 * deg.clamp(min=1).sqrt().unsqueeze(1)
        errM = c * (absk + k * (mu.abs() + mmax) * absk1) * U
        # where M_k is within its rounding error of 0, fp32 may see rho_k at its largest, (1/k) 1e-5^(1/k - 1), where float64
        # sees 0 (exactly symmetric neighbourhoods): bound with the largest
        rho = torch.where(M.abs() <= errM, torch.full_like(M, (1.0 / k) * EPS ** (1.0 / k - 1.0)),
                          (1.0 / k) * (M.abs() + EPS) ** (1.0 / k - 1.0))
        drho = (1.0 / k) * abs(1.0 / k - 1.0) * (M.abs() + EPS) ** (1.0 / k - 2.0)
        a = G[k].double().abs() * k / cnt
        absk2 = torch.zeros_like(mu).index_add(0, dst, delta.abs() ** (k - 2)) / cnt
        shape = delta.abs() ** (k - 1) + C.abs()[dst]
        # the roundings of delta_j^(k-1) and of C_(k-1) (a sum of mixed signs: its error scales with sum |delta|^(k-1)), and
        # the error of mu / delta carried through both
        spread = delta.abs() ** (k - 1) + absk1[dst] + \
            (k - 1) * (mu.abs() + mmax)[dst] * (delta.abs() ** (k - 2) + absk2[dst])
        t1 = (a * rho)[dst] * spread * c[dst] * U
        t2 = (a * drho * errM)[dst] * shape
        tol = tol + t1 + t2
    return g64, scale * tol
