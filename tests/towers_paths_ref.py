"""numpy restatement of the tower post linear (k_towers_3xtf32 in pna_b200/csrc/pna_linear.cu) -- TEST INFRASTRUCTURE.

Per tower t the kernel runs a 3xTF32 product over a VIRTUAL K axis that its loaders gather, padded with zeros to a
multiple of 32:
  * forward (pna_linear_towers_scaled_fwd): x' = [self_t | fl(c_0 agg_t) | .. | fl(c_{S-1} agg_t)], the reference
    weight W_t [O_t, (1 + S A) Fp] read as it is;
  * data gradient (pna_linear_towers_bwd_data): x' = [dY_t | fl(c_0 dY_t) | .. | fl(c_{S-1} dY_t)] against
    W''[c, k]: k < O_t -> W_t[k, c] for the self columns c < Fp (else 0); k = O_t + s O_t + o -> W_t[o, Fp + s A Fp + c - Fp]
    for the aggregate columns c >= Fp (else 0).
The chains restart every kLinFoldSteps K blocks, in both directions, and are folded as linear_paths_ref.linear_restate
states it (the bias after the last block).  Operands, chains and bars come from linear_paths_ref.
"""
from __future__ import annotations

import numpy as np

from linear_paths_ref import F32, LIN_BK, LIN_FOLD_STEPS, grid_matrix, grid_scales, linear_restate, rounding_slack, split, \
    chain_budget, _groups


def _pad_k(m):
    return np.pad(m, ((0, 0), (0, (-m.shape[1]) % LIN_BK)))


def _scaled(x, c):
    with np.errstate(invalid="ignore", over="ignore"):
        return [np.asarray(x, F32) * c[:, s:s + 1].astype(F32) for s in range(c.shape[1])]


def fwd_operands(a, c, w, t, fp, n_aggr):
    """(x' [N, Kv32], W_t [O_t, Kv32]) of tower t."""
    per = (1 + n_aggr) * fp
    a_t = np.asarray(a, F32)[:, t * per:(t + 1) * per]
    x = np.concatenate([a_t[:, :fp]] + _scaled(a_t[:, fp:], c), axis=1)
    return _pad_k(x), _pad_k(np.asarray(w[t], F32))


def bwd_operands(gy, c, w, t, fp, n_aggr):
    """(x' [N, Kv32], W'' [(1 + A) Fp, Kv32]) of tower t."""
    _, o, kw = w.shape
    af, s_n = n_aggr * fp, c.shape[1]
    g_t = np.asarray(gy, F32)[:, t * o:(t + 1) * o]
    x = np.concatenate([g_t] + _scaled(g_t, c), axis=1)
    wt = np.asarray(w[t], F32)
    wr = np.zeros((fp + af, (1 + s_n) * o), F32)
    wr[:fp, :o] = wt[:, :fp].T
    for s in range(s_n):
        wr[fp:, (1 + s) * o:(2 + s) * o] = wt[:, fp + s * af:fp + (s + 1) * af].T
    return _pad_k(x), _pad_k(wr)


def fwd_restate(a, c, w, b, fp, n_aggr, bars=False, fold=LIN_FOLD_STEPS, lolo=False):
    """y [N, T O_t] (and its elementwise bar on random data)."""
    t_n = w.shape[0]
    ys, brs = [], []
    for t in range(t_n):
        x, wt = fwd_operands(a, c, w, t, fp, n_aggr)
        xh, xl = split(x)
        wh, wl = split(wt)
        r = linear_restate(xh, xl, wh, wl, None if b is None else np.asarray(b[t], F32), fold, lolo, bars)
        ys.append(r[0] if bars else r)
        if bars:
            brs.append(r[1] + rounding_slack(r[0], 2 + x.shape[1] // (LIN_BK * LIN_FOLD_STEPS)))
    y = np.concatenate(ys, axis=1)
    return (y, np.concatenate(brs, axis=1)) if bars else y


def bwd_restate(gy, c, w, fp, n_aggr, bars=False, fold=LIN_FOLD_STEPS, lolo=False):
    """grad_a [N, T (1 + A) Fp] (and its bar)."""
    t_n = w.shape[0]
    gs, brs = [], []
    for t in range(t_n):
        x, wr = bwd_operands(gy, c, w, t, fp, n_aggr)
        xh, xl = split(x)
        wh, wl = split(wr)
        r = linear_restate(xh, xl, wh, wl, None, fold, lolo, bars)
        gs.append(r[0] if bars else r)
        if bars:
            brs.append(r[1] + rounding_slack(r[0], 2 + x.shape[1] // (LIN_BK * LIN_FOLD_STEPS)))
    g = np.concatenate(gs, axis=1)
    return (g, np.concatenate(brs, axis=1)) if bars else g


def budget(kind, x1, c, w, fp, n_aggr):
    """Largest sum|terms| / u over the chains of every tower (exact tier: <= 2^12)."""
    worst = 0.0
    for t in range(w.shape[0]):
        x, wt = (fwd_operands if kind == "fwd" else bwd_operands)(x1, c, w, t, fp, n_aggr)
        xh, xl = split(x)
        wh, wl = split(wt)
        worst = max(worst, chain_budget(xh, xl, wh, wl, _groups(x.shape[1] // LIN_BK, LIN_FOLD_STEPS)))
    return worst


# (n, T, Fp, O_t, A, S): N = 1, N not a multiple of 128, K not a multiple of 32 (ZINC: (1 + 4) 16 = 80), O_t not a multiple of 8
CASES = [
    (1, 1, 16, 14, 1, 2),
    (129, 2, 32, 15, 4, 3),
    (200, 4, 16, 32, 4, 3),      # the ZINC tower block
    (130, 5, 16, 14, 4, 3),      # the DGL ZINC layer (70 / 5 towers)
    (257, 4, 32, 32, 4, 3),      # PNAConv(128, 128, towers=4, divide_input=True)
    (100, 1, 64, 64, 6, 5),
    (64, 2, 76, 20, 6, 2),
    (300, 4, 64, 16, 1, 5),
    (131, 5, 76, 15, 4, 3),
]


def case_data(case, grid=True, seed=0):
    """(a, c, w, b, gy, deg0 rows): grid operands (exact tier) or random ones.  Rows with c = 0 in their scaled copies stand
    for in-degree 0 (amplification of an isolated row); their aggregate blocks are zero, as the aggregation writes them."""
    n, t_n, fp, o, n_aggr, s_n = case
    rng = np.random.default_rng(seed + n + 7 * t_n + fp + o + n_aggr + s_n)
    per, kw = (1 + n_aggr) * fp, (1 + s_n * n_aggr) * fp
    if grid:
        dens_a = min(0.9, 60.0 / min(kw, LIN_FOLD_STEPS * LIN_BK))
        ah, al = grid_matrix(rng, (n, t_n * per), -3, dens_a)
        wh, wl = grid_matrix(rng, (t_n * o, kw), -4, min(0.9, 60.0 / min(kw, LIN_FOLD_STEPS * LIN_BK)), lo_shift=19)
        yh, yl = grid_matrix(rng, (n, t_n * o), -3, min(0.9, 60.0 / min((1 + s_n) * o, LIN_FOLD_STEPS * LIN_BK)))
        a, w, gy = ah + al, (wh + wl).reshape(t_n, o, kw), yh + yl
        c = grid_scales(rng, n, s_n)
        b = (rng.integers(-3, 4, (t_n, o)) * 2.0 ** -10).astype(F32)
    else:
        a = rng.standard_normal((n, t_n * per)).astype(F32)
        w = (rng.standard_normal((t_n, o, kw)) / np.sqrt(kw)).astype(F32)
        gy = rng.standard_normal((n, t_n * o)).astype(F32)
        c = rng.uniform(0.2, 2.5, (n, s_n)).astype(F32)
        c[:, 0] = 1.0
        b = rng.standard_normal((t_n, o)).astype(F32)
    iso = np.arange(n) % 7 == 3
    for t in range(t_n):
        a[iso, t * per + fp:(t + 1) * per] = 0
    c[iso, 1:] = 0
    return a, c, w, b, gy
