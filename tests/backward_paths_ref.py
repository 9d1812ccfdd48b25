"""fp32 restatement of pna_aggregate_bwd for sum / mean / min / max / var / std -- TEST INFRASTRUCTURE (CPU only).

The backward (pna_b200/csrc/pna_aggregate_bwd.cu) is built with -fmad=false and rounds every operation on its own, so each
step below is one numpy float32 operation in the kernel's order:
  * row_stats_bwd: pass A per row in CSR slot order (sum += m; sq += fl(m*m); strict < / > keeps the FIRST arg slot).  Split
    rows (deg >= split_threshold) are reduced per chunk of `chunk_edges` slots and the chunk partials are merged
    SEQUENTIALLY in chunk order, as k_bwd_hub_coef does -- not the forward's two-level or radix-tree order.
  * coefficients: (c0, c1, gmin, gmax) per row and feature from grad_out; the degree-scaler factors are an input (the
    library's own, pna_row_scales), never recomputed with a host logarithm.
  * slot_grads: grad_m = ((c0 + c1*m) + [argmin] gmin) + [argmax] gmax per slot, grad_row_bias summed in slot order (split
    rows: per-chunk shares, each in slot order, added in chunk order -- the per-slot instance's k_bwd_hub_bias).
  * coef_rows / routed_terms / combine: the coefficient mode (pna_aggregate_bwd_coef, pna_aggregate_bwd_combine).
  * order_free_sum: the sums the atomics form, as a float64 value with a rigorous per-element bound.
A message is m = fl(x[col[slot]] + bias[row]) with a row bias; bf16 inputs are widened to fp32 exactly first.
"""
from __future__ import annotations

import numpy as np

import forward_paths_ref as FR

F32 = np.float32
F64 = np.float64
U32 = 2.0 ** -24        # unit roundoff of fp32
U64 = 2.0 ** -53
EPS_STD = F32(1e-5)


# ---- which instance bwd_entry launches (vec_ok, launch_bwd_typed, launch_bwd) ---------------------------------------------
def bwd_vec_ok(ft: int, elem_bytes: int, rows) -> bool:
    """bwd_entry's vec_ok: Ft a multiple of the 16-byte vector, and every (address, pitch in elements) of gathered, grad_out
    and row_bias (when given) 16-byte aligned / a multiple of the vector."""
    vec = 16 // elem_bytes
    return ft % vec == 0 and all(addr % 16 == 0 and pitch % vec == 0 for addr, pitch in rows)


def bwd_instance(width: int, elem_bytes: int, vec_ok: bool) -> tuple:
    """(VEC, G, gridDim.y) of launch_bwd_typed / launch_bwd for `width` columns (n_feat, or the slab's f_count)."""
    vec = 16 // elem_bytes if vec_ok else 1
    chunks = width // vec
    g = next((g for g in (1, 2, 4, 8, 16) if chunks <= g), 32)
    return vec, g, -(-width // (g * vec))


# ---- pass A --------------------------------------------------------------------------------------------------------------
def _messages(x, col, slots, bias, rows):
    m = x[slots if col is None else col[slots]]
    return m + bias[rows] if bias is not None else m


def _segments(x, col, beg, length, bias, rows):
    """(sum, sq, mn, mx, amn, amx) of R slot segments [beg, beg + length), slot by slot; arg slots absolute, -1 = none."""
    R, F = len(beg), x.shape[1]
    s, q = np.zeros((R, F), F32), np.zeros((R, F), F32)
    mn, mx = np.full((R, F), np.inf, F32), np.full((R, F), -np.inf, F32)
    amn, amx = np.full((R, F), -1, np.int64), np.full((R, F), -1, np.int64)
    beg, length = np.asarray(beg, np.int64), np.asarray(length, np.int64)
    for k in range(int(length.max()) if R else 0):
        a = np.nonzero(length > k)[0]
        slot = beg[a] + k
        m = _messages(x, col, slot, bias, rows[a])
        s[a] = s[a] + m
        q[a] = q[a] + m * m
        lt, gt = m < mn[a], m > mx[a]
        mn[a] = np.where(lt, m, mn[a])
        amn[a] = np.where(lt, slot[:, None], amn[a])
        mx[a] = np.where(gt, m, mx[a])
        amx[a] = np.where(gt, slot[:, None], amx[a])
    return [s, q, mn, mx, amn, amx]


def chunk_bounds(rowptr, hub_info, chunk_edges):
    """(row, begin, length) of every chunk of every split row, split row by split row, chunks in order."""
    rows, beg, ln = [], [], []
    for r, _, nch, d in hub_info:
        j = np.arange(nch)
        rows.append(np.full(nch, r))
        beg.append(rowptr[r] + j * chunk_edges)
        ln.append(np.minimum(chunk_edges, d - j * chunk_edges))
    cat = (lambda v: np.concatenate(v).astype(np.int64)) if rows else (lambda v: np.zeros(0, np.int64))
    return cat(rows), cat(beg), cat(ln)


def row_stats_bwd(x, rowptr, col, hub_info, chunk_edges, bias=None):
    """[sum, sq, mn, mx, amn, amx], each [N, F]: pass A of k_bwd_rows, or k_bwd_hub_stats + the sequential chunk-order merge
    of k_bwd_hub_coef for split rows (fl32 adds starting from 0; strict < / >, so a tie in a later chunk keeps the earlier
    chunk's slot)."""
    N = len(rowptr) - 1
    deg = np.diff(rowptr)
    light = deg.copy()
    light[hub_info[:, 0]] = 0
    st = _segments(x, col, rowptr[:-1], light, bias, np.arange(N))
    crow, cbeg, clen = chunk_bounds(rowptr, hub_info, chunk_edges)
    P = _segments(x, col, cbeg, clen, bias, crow)
    c = 0
    for r, _, nch, _ in hub_info:
        acc = [a[r] for a in st]            # the row's light statistics are the initial values (0, 0, inf, -inf, -1, -1)
        for j in range(c, c + nch):
            acc[0] = acc[0] + P[0][j]
            acc[1] = acc[1] + P[1][j]
            lt, gt = P[2][j] < acc[2], P[3][j] > acc[3]
            acc[2], acc[4] = np.where(lt, P[2][j], acc[2]), np.where(lt, P[4][j], acc[4])
            acc[3], acc[5] = np.where(gt, P[3][j], acc[3]), np.where(gt, P[5][j], acc[5])
        for a, v in zip(st, acc):
            a[r] = v
        c += nch
    return st


# ---- coefficients -------------------------------------------------------------------------------------------------------
def coefficients(st, deg, grad_out, scales, aggrs, *, towers=1, has_self=False, relu_var=False):
    """(c0, c1, gmin, gmax), each [N, F] float32.  grad_out [N, >= T*Wt] (fp32 values), scales [N, S] fp32 (the scalers'
    factors for the degree the kernel sees: pna_row_scales of the in-degree, or of scaler_degree).  aggrs may contain
    "_skip" (PNA_AGGR_SKIP) entries, which take their column slot and add nothing."""
    s_sum, s_sq = st[0], st[1]
    N, F = s_sum.shape
    S, A = scales.shape[1], len(aggrs)
    Ft = F // towers
    Wt = (int(has_self) + A * S) * Ft
    f = np.arange(F)
    ooff = (f // Ft) * Wt + int(has_self) * Ft + f % Ft
    cnt = np.maximum(np.asarray(deg), 1).astype(F32)[:, None]
    mean = s_sum / cnt
    var = s_sq / cnt - mean * mean
    sd = np.sqrt(np.maximum(var, F32(0)) + EPS_STD)
    go = np.asarray(grad_out, F32)
    scales = np.asarray(scales, F32)
    c0, c1, gmin, gmax = (np.zeros((N, F), F32) for _ in range(4))
    for a, name in enumerate(aggrs):
        if name == "_skip":
            continue
        g = np.zeros((N, F), F32)
        for s in range(S):
            g = g + scales[:, s:s + 1] * go[:, ooff + (s * A + a) * Ft]
        if name == "sum":
            c0 = c0 + g
        elif name == "mean":
            c0 = c0 + g / cnt
        elif name == "min":
            gmin = gmin + g
        elif name == "max":
            gmax = gmax + g
        elif name in ("var", "std"):
            if name == "var":
                t = F32(2) * g / cnt
                if relu_var:
                    t = np.where(var > 0, t, F32(0))
            else:
                t = np.where(var > 0, g / (cnt * sd), F32(0))
            c1 = c1 + t
            c0 = c0 - t * mean
        else:
            raise ValueError(f"{name}: not restated here (moments and weighted aggregators have their own oracles)")
    return c0, c1, gmin, gmax


# ---- pass C -------------------------------------------------------------------------------------------------------------
def ordered_sums(vals, beg, length):
    """[R, F]: fp32 sums of vals[beg[r] : beg[r] + length[r]] in slot order, starting from 0."""
    R = len(beg)
    out = np.zeros((R, vals.shape[1]), F32)
    beg, length = np.asarray(beg, np.int64), np.asarray(length, np.int64)
    for k in range(int(length.max()) if R else 0):
        a = np.nonzero(length > k)[0]
        out[a] = out[a] + vals[beg[a] + k]
    return out


def slot_rows(rowptr):
    return np.repeat(np.arange(len(rowptr) - 1), np.diff(rowptr))


def slot_grads(c, st, x, rowptr, col, hub_info, chunk_edges, bias=None):
    """(grad_m [E, F], grad_row_bias [N, F], chunk_shares [C, F]).  grad_row_bias is the per-slot instance's: light rows sum
    their slots in order, split rows add their chunks' shares (each in slot order) in chunk order; isolated rows get 0.
    The atomic instance adds split rows' shares in any order: check it with order_free_sum over chunk_shares."""
    c0, c1, gmin, gmax = c
    amn, amx = st[4], st[5]
    row = slot_rows(rowptr)
    slot = np.arange(len(row))
    m = _messages(x, col, slot, bias, row)
    gm = c0[row] + c1[row] * m
    gm = gm + np.where(amn[row] == slot[:, None], gmin[row], F32(0))
    gm = gm + np.where(amx[row] == slot[:, None], gmax[row], F32(0))
    deg = np.diff(rowptr)
    light = deg.copy()
    light[hub_info[:, 0]] = 0
    gb = ordered_sums(gm, rowptr[:-1], light)
    _, cbeg, clen = chunk_bounds(rowptr, hub_info, chunk_edges)
    shares = ordered_sums(gm, cbeg, clen)
    c = 0
    for r, _, nch, _ in hub_info:
        acc = np.zeros(gm.shape[1], F32)
        for j in range(c, c + nch):
            acc = acc + shares[j]
        gb[r] = acc
        c += nch
    return gm, gb, shares


# ---- coefficient mode ---------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """Correctly rounded fp32 fma(a, b, c): a*b is exact in float64; the float64 sum with its TwoSum error is rounded to odd
    (53 >= 24 + 2 bits, so the final cast to fp32 rounds once, correctly).  Plain float64 a*b + c double-rounds."""
    a, b, c = (np.asarray(v, F32).astype(F64) for v in (a, b, c))
    p = a * b
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))
    even = (s.view(np.uint64) & np.uint64(1)) == 0
    s = np.where((err != 0) & even, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


def coef_rows(c, st, deg, bias=None):
    """(c0', c1, grad_row_bias) of emit_row: c0' = fma(c1, bias, c0) (c0 without a bias) and the closed form
    grad_row_bias = ((deg*c0 + c1*sum) + gmin) + gmax, with deg*c0 one fp32 multiply."""
    c0, c1, gmin, gmax = c
    c0p = fma32(c1, bias, c0) if bias is not None else c0.copy()
    degf = np.asarray(deg).astype(F32)[:, None]
    gb = ((degf * c0 + c1 * st[0]) + gmin) + gmax
    return c0p, c1, gb


def routed_terms(c, st, deg, col):
    """(source row, feature, value) of the min / max atomics of emit_row: gmin to the source of the argmin slot, gmax to that
    of the argmax slot, where the gradient is nonzero (rows without in-edges emit nothing)."""
    rows, feats, vals = [], [], []
    has = (np.asarray(deg) > 0)[:, None]
    for g, arg in ((c[2], st[4]), (c[3], st[5])):
        r, f = np.nonzero(has & (g != 0) & (arg >= 0))
        rows.append(col[arg[r, f]])
        feats.append(f)
        vals.append(g[r, f])
    return np.concatenate(rows), np.concatenate(feats), np.concatenate(vals).astype(F32)


def combine(gg, s0, s1, x):
    """k_bwd_combine: gg = fl(gg + fl(s0 + fl(x*s1)))."""
    return gg + (s0 + x * s1)


def transposed_sums(vals, host_t, chunk_edges, width_for_launch, vec_ok):
    """The forward 'sum' of vals [n_dst, W] over a transposed CSR (host arrays rowptr, col, hub_info, chunk_items), merged
    the way pna_aggregate_fwd merges that CSR's split rows at this width (forward_paths_ref.merge_kind)."""
    rowptr, col, info, items = host_t
    G = FR.lane_group(width_for_launch, 4, vec_ok)[0]
    deg = np.diff(rowptr)
    merge = FR.merge_kind(int(deg.max()) if deg.size else 0, chunk_edges, G)
    return FR.row_stats(vals, rowptr, col, info, items, chunk_edges, merge)[:, 0], merge


# ---- order-free sums (atomics) ------------------------------------------------------------------------------------------
def order_free_sum(n_rows, rows, terms):
    """(float64 sum [n_rows, F], bound [n_rows, F]) of the fp32 terms [K, F] added into row rows[k] (from 0) in ANY order:
    a float32 sum of k terms lies within gamma_{k-1} * sum |t| of the exact sum (gamma_n = n u / (1 - n u), u = 2^-24); the
    float64 evaluation of the exact sum adds its own gamma_{k-1} (u = 2^-53).  Their total is a rigorous per-element bar."""
    rows = np.asarray(rows, np.int64)
    terms = np.asarray(terms, F32)
    F = terms.shape[1]
    s, a = np.zeros((n_rows, F), F64), np.zeros((n_rows, F), F64)
    k = np.bincount(rows, minlength=n_rows).astype(F64)
    if rows.size:
        order = np.argsort(rows, kind="stable")
        r_sorted = rows[order]
        starts = np.nonzero(np.r_[True, r_sorted[1:] != r_sorted[:-1]])[0]
        t = terms[order].astype(F64)
        s[r_sorted[starts]] = np.add.reduceat(t, starts, axis=0)
        a[r_sorted[starts]] = np.add.reduceat(np.abs(t), starts, axis=0)
    km1 = np.maximum(k - 1, 0)[:, None]
    bound = (km1 * U32 / (1 - km1 * U32) + km1 * U64 / (1 - km1 * U64)) * a
    return s, bound


def order_free_sum_elements(shape, rows, feats, vals, base=None):
    """order_free_sum for scattered scalar terms: vals[k] added into element (rows[k], feats[k]), plus (optionally) one term
    base[r, f] into every element -- the coefficient path's routed min / max atomics followed by k_bwd_combine's addend."""
    s, a, k = np.zeros(shape, F64), np.zeros(shape, F64), np.zeros(shape, F64)
    v = np.asarray(vals, F64)
    np.add.at(s, (rows, feats), v)
    np.add.at(a, (rows, feats), np.abs(v))
    np.add.at(k, (rows, feats), 1.0)
    if base is not None:
        s, a, k = s + np.asarray(base, F64), a + np.abs(np.asarray(base, F64)), k + 1
    km1 = np.maximum(k - 1, 0)
    return s, (km1 * U32 / (1 - km1 * U32) + km1 * U64 / (1 - km1 * U64)) * a, k


def within_order_free(got, s, bound):
    """boolean [n, F]: got lies within the bound of the float64 sum"""
    return np.abs(np.asarray(got, F64) - s) <= bound
