"""Error bars of the slot-weighted aggregation (pna_aggregate_fwd_weighted) against float64 of the same formula on the same fp32
messages, derived the way tests/weighted_bars.py derives its own: one term u = 2^-24 per rounding, a slot-order sum of d
terms growing like sqrt(d) (rounding errors of random sign), a safety factor K = 4.

For row i with slots s (messages m_s, weights w_s, d slots):
  W    = sum w_s                      e_W = u sqrt(d) sum |w_s|
  S    = sum fl(m_s w_s)              e_S = u (1 + sqrt(d)) sum |m_s w_s|              (product, then the sum)
  Q    = sum fl(fl(m_s m_s) w_s)      e_Q = u (2 + sqrt(d)) sum m_s^2 |w_s|
  mean = S / W                        e_mean = u |mean| + (e_S + |mean| e_W) / |W|
  var  = Q / W - mean^2               e_var  = u |Q/W| + (e_Q + |Q/W| e_W) / |W| + 2 |mean| e_mean + u mean^2 + u |var|
  std  = sqrt(max(var, 0) + 1e-5)     e_std  = e_var / (2 std) + u std
  min / max: exact.  A scaler multiplies once more: + u |y s|, and the factor itself is within 2u.
Gradient of slot s (upstream G_a per aggregator, identity scaler): the float64 value of w_s (c0 + c1 m_s) + routed terms, held
term by term: each aggregator's term gets the relative error of its coefficient (the divisions by W, by W std, the
cancellation of c0 + c1 m = t (m - mean)) plus the two roundings of the slot formula."""
import math

import torch

U = 2.0 ** -24
K = 4.0


def row_sums(msg, w, dst, n):
    """float64 per-row sums: W, S, Q, sum|w|, sum|m w|, sum m^2|w|, d  ([n] or [n, F])."""
    m, w = msg.double(), w.double()
    F = m.size(1)
    z = lambda: torch.zeros(n, F, dtype=torch.float64)
    W = torch.zeros(n, dtype=torch.float64).index_add(0, dst, w)
    Wabs = torch.zeros(n, dtype=torch.float64).index_add(0, dst, w.abs())
    d = torch.bincount(dst, minlength=n).double()
    S = z().index_add(0, dst, m * w[:, None])
    Sabs = z().index_add(0, dst, (m * w[:, None]).abs())
    Q = z().index_add(0, dst, m * m * w[:, None])
    Qabs = z().index_add(0, dst, m * m * w.abs()[:, None])
    return W, S, Q, Wabs, Sabs, Qabs, d


def forward(msg, w, dst, n):
    """{aggregator: (float64 value, bar)} of the weighted aggregation, rows with slots (others: value 0, bar 0 except std)."""
    W, S, Q, Wabs, Sabs, Qabs, d = row_sums(msg, w, dst, n)
    sq = d.sqrt()[:, None]
    Wc = W[:, None]
    eW = U * sq * Wabs[:, None]
    eS = U * (1 + sq) * Sabs
    eQ = U * (2 + sq) * Qabs
    mean = S / Wc
    emean = U * mean.abs() + (eS + mean.abs() * eW) / Wc.abs()
    q = Q / Wc
    var = q - mean * mean
    evar = U * q.abs() + (eQ + q.abs() * eW) / Wc.abs() + 2 * mean.abs() * emean + U * mean * mean + U * var.abs()
    std = (var.clamp(min=0) + 1e-5).sqrt()
    estd = evar / (2 * std) + U * std
    m = msg.double()
    pos = w > 0
    big = torch.full((n, m.size(1)), -math.inf, dtype=torch.float64)
    mx = big.index_reduce(0, dst[pos], m[pos], "amax", include_self=True)
    mn = (-big).index_reduce(0, dst[pos], m[pos], "amin", include_self=True)
    none = torch.isinf(mx)
    mx, mn = torch.where(none, 0.0, mx), torch.where(none, 0.0, mn)
    iso = (d == 0)[:, None]
    out = dict(sum=(S, eS), mean=(mean, emean), var=(var.clamp(min=0), evar), std=(std, estd), max=(mx, 0 * mx), min=(mn, 0 * mn))
    res = {}
    for k, (v, e) in out.items():
        v = torch.where(iso, torch.full_like(v, math.sqrt(1e-5) if k == "std" else 0.0), v)
        e = torch.where(iso, 2 * U * v.abs(), e)           # isolated rows: the constant sqrt(1e-5) of std, rounded
        res[k] = (v, K * e)
    return res


def scaled_bar(y, bar, fac):
    """value and bar of a scaled column: fl(y * fac), fac within 2u."""
    v = y * fac
    return v, bar * fac.abs() + K * 3 * U * v.abs()


def slot_grads(msg, w, dst, n, G, relu_var=True):
    """float64 per-slot gradients [E, F] (edge order) and their bars, identity scaler; G = {aggregator: [n, F] upstream}.
    min / max route to the first slot (edge order) attaining the extremum among the positive weights."""
    W, S, Q, Wabs, Sabs, Qabs, d = row_sums(msg, w, dst, n)
    f = forward(msg, w, dst, n)
    m, wd = msg.double(), w.double()[:, None]
    Wc = W[:, None]
    mean, emean = f["mean"][0], f["mean"][1] / K
    var = Q / Wc - mean * mean
    std = (var.clamp(min=0) + 1e-5).sqrt()
    g = torch.zeros_like(m)
    bar = torch.zeros_like(m)
    rel_W = U * d.sqrt()[:, None] * Wabs[:, None] / Wc.abs()
    for name, Gr in G.items():
        Gr = Gr.double()
        Gs = Gr[dst]
        if name == "sum":
            term = wd * Gs
            tb = 2 * U * term.abs()
        elif name == "mean":
            term = wd * Gs / Wc[dst]
            tb = term.abs() * (3 * U + rel_W[dst])
        elif name in ("var", "std"):
            if name == "var":
                t = 2 * Gr / Wc
                if relu_var:
                    t = torch.where(var > 0, t, 0.0)
                rel_t = 3 * U + rel_W
            else:
                t = torch.where(var > 0, Gr / (Wc * std), 0.0)
                rel_t = 4 * U + rel_W + (f["std"][1] / K) / std
            dm = m - mean[dst]
            term = wd * t[dst] * dm
            # c0 + c1 m = t m - t mean: cancellation, each product and the sum rounded
            tb = (wd * t[dst]).abs() * (dm.abs() * rel_t[dst] + emean[dst] + 3 * U * (m.abs() + mean[dst].abs()))
            # var within its bar of 0 (one slot, equal messages): the fp32 mask [var > 0] may differ from float64's, and the
            # kernel's term is then t' (m - mean) evaluated in fp32 with t' the largest coefficient var >= 0 allows
            amb = f["var"][1] / K >= var.abs()
            t_amb = (2 * Gr / Wc).abs() if name == "var" else (Gr / (Wc * math.sqrt(1e-5))).abs()
            tb_amb = wd.abs() * t_amb[dst] * (dm.abs() + emean[dst] + 3 * U * (m.abs() + mean[dst].abs()))
            tb = torch.where(amb[dst], torch.maximum(tb, tb_amb), tb)
        else:
            pos = (w > 0)
            key = m if name == "max" else -m
            best = torch.full((n, m.size(1)), -math.inf, dtype=torch.float64).index_reduce(0, dst[pos], key[pos], "amax")
            hit = pos[:, None] & (key == best[dst])
            first = torch.zeros_like(hit)
            seen = torch.zeros(n, m.size(1), dtype=torch.bool)
            for e in range(m.size(0)):          # first slot in CSR (= stable edge) order
                r = dst[e]
                first[e] = hit[e] & ~seen[r]
                seen[r] |= hit[e]
            term = torch.where(first, Gs, 0.0)
            tb = 2 * U * term.abs()
        g, bar = g + term, bar + tb
    return g, K * (bar + U * g.abs())
