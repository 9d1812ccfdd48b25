"""fp32 restatement of the add-on aggregators, forward and backward -- TEST INFRASTRUCTURE (CPU only).

moment3 / moment4 / moment5 (pna_b200/csrc/pna_aggregate_moments.cuh) and softmax / softmin / normalised_mean
(pna_aggregate_weighted.cuh) are built with -fmad=false and round every operation on their own, in the order their headers
spell out, so each step below is one numpy float32 operation in the kernel's order:
  * messages: m = fl(x[src] + bias[row]); src = col[slot], or the slot itself when col is None (messages in CSR order);
    bf16 inputs and grad_out are widened to fp32 exactly by the caller.
  * row sums: light rows (deg < split_threshold) add their slots in order from 0; split rows add each chunk of
    `chunk_edges` slots in order from 0, then the chunk sums in chunk order from 0.
  * quotients by the in-degree are correctly rounded (IEEE division); D^(-1/2) is the correctly rounded reciprocal square
    root (the float64 value rounded once: the same float for every D < 2^22).
  * powf and expf are the only roundings nobody states: they are injected (`DevMath`), as libm's functions on the host and
    the device's own bits (oracle/devmath) on the GPU.  Every argument is computed here, exactly in fp32.
  * scaler factors are an input ([N, S], the library's pna_row_scales at the scalers' degree), never a host logarithm.
The backward composes with backward_paths_ref: the core kernel STORES its term (add-on codes as PNA_AGGR_SKIP), then the
add-on families ADD theirs in launch order: moments, then softmax, softmin, normalised_mean (code order, whatever the
list order).  grad_row_bias: the core writes it, each family adds its row sum (light rows: slot order; split rows: the chunk
shares in chunk order, k_mom_bwd_hub_bias).
"""
from __future__ import annotations

import ctypes
import ctypes.util

import numpy as np

import backward_paths_ref as B

F32 = np.float32
MOMENTS = {"moment3": 3, "moment4": 4, "moment5": 5}
WEIGHTED = ("softmax", "softmin", "normalised_mean")   # codes 9, 10, 11: the launch order
INV_K = {3: F32(1) / F32(3), 4: F32(0.25), 5: F32(0.2)}                  # moment_inv: 1.0f / 3.0f, 0.25f, 0.2f
SLOPE_E = {3: F32(F32(1) / F32(3)) - F32(1), 4: F32(-0.75), 5: F32(-0.8)}  # moment_slope: (1.0f/3.0f - 1.0f), -0.75f, -0.8f
EPS = F32(1e-5)
FLAG_ZERO_ISOLATED, FLAG_SKIP_LIGHT, FLAG_SKIP_HUBS = 1, 2, 4
MOM_THREADS = 256                                                          # kMomThreads: 8 rows or chunks per CTA


# ---- injected device math ---------------------------------------------------------------------------------------------
class DevMath:
    """powf(x, y) and expf(x) over float32 arrays (elementwise, same shape)."""

    def __init__(self, powf, expf, name):
        self._powf, self._expf, self.name = powf, expf, name

    def powf(self, x, y):
        x = np.ascontiguousarray(x, F32)
        y = np.ascontiguousarray(np.broadcast_to(np.asarray(y, F32), x.shape), F32)
        return np.asarray(self._powf(x, y), F32).reshape(x.shape) if x.size else x.copy()

    def expf(self, x):
        x = np.ascontiguousarray(x, F32)
        return np.asarray(self._expf(x), F32).reshape(x.shape) if x.size else x.copy()


def host_math() -> DevMath:
    """libm's powf / expf through ctypes: what the host build of the kernels (tests/emu) calls."""
    libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
    libm.powf.restype, libm.powf.argtypes = ctypes.c_float, [ctypes.c_float, ctypes.c_float]
    libm.expf.restype, libm.expf.argtypes = ctypes.c_float, [ctypes.c_float]

    def powf(x, y):
        return np.array([libm.powf(float(a), float(b)) for a, b in zip(x.ravel(), y.ravel())], F32)

    def expf(x):
        return np.array([libm.expf(float(a)) for a in x.ravel()], F32)
    return DevMath(powf, expf, "libm")


def div(x, d):
    """correctly rounded fp32 quotient x / d (d: integer per row, broadcast over features)"""
    return np.asarray(x, F32) / np.asarray(d).astype(F32)[:, None]


def rsqrt_deg(D):
    """D^(-1/2) correctly rounded, 0 for D == 0 (wsum_rsqrt / wsum_rsqrt_deg)"""
    D = np.asarray(D, np.float64)
    return np.where(D > 0, 1.0 / np.sqrt(np.maximum(D, 1.0)), 0.0).astype(F32)


# ---- graph layout ------------------------------------------------------------------------------------------------------
class Graph:
    """The CSR the kernels see (host arrays): rowptr [N+1], col [E] or None (messages in CSR order), hub_info [H, 4] =
    (row, first chunk, n chunks, degree) in the GPU's hub order, chunk_edges, split_threshold, and degree_col [E] or None."""

    def __init__(self, rowptr, col, hub_info, chunk_edges, split, dcol=None):
        self.rowptr = np.asarray(rowptr, np.int64)
        self.col = None if col is None else np.asarray(col, np.int64)
        self.hub_info = np.asarray(hub_info, np.int64).reshape(-1, 4)
        self.chunk, self.split = int(chunk_edges), int(split)
        self.dcol = None if dcol is None else np.asarray(dcol, np.int64)
        self.n = len(self.rowptr) - 1
        self.deg = np.diff(self.rowptr)
        self.row = B.slot_rows(self.rowptr)
        self.hub = np.zeros(self.n, bool)
        self.hub[self.hub_info[:, 0]] = True
        self.light_len = np.where(self.hub, 0, self.deg)
        self.crow, self.cbeg, self.clen = B.chunk_bounds(self.rowptr, self.hub_info, self.chunk)

    def messages(self, x, bias):
        slot = np.arange(len(self.row))
        m = x[slot if self.col is None else self.col]
        return m + bias[self.row] if bias is not None else m

    def row_sums(self, vals):
        """([N, F] per-row fp32 sums as the kernels form them, [C, F] chunk sums); rows of neither kind hold 0."""
        s = B.ordered_sums(vals, self.rowptr[:-1], self.light_len)
        shares = B.ordered_sums(vals, self.cbeg, self.clen)
        c = 0
        for r, _, nch, _ in self.hub_info:
            acc = np.zeros(vals.shape[1], F32)
            for j in range(c, c + nch):
                acc = acc + shares[j]
            s[r] = acc
            c += nch
        return s, shares

    def row_max(self, vals):
        """[N, F] fmaxf over each row's slots from -inf (exact: chunk maxima merged give the same value)"""
        out = np.full((self.n, vals.shape[1]), -np.inf, F32)
        nz = self.deg > 0
        if nz.any():
            out[nz] = np.fmax(np.fmax.reduceat(vals, self.rowptr[:-1][nz], axis=0), out[nz])
        return out

    def degree_node(self):
        """the node whose degree weighs each slot: degree_col, else col"""
        return self.dcol if self.dcol is not None else self.col


# ---- per-row quantities ------------------------------------------------------------------------------------------------
def central(g: Graph, m):
    """(mu [N, F], delta^2..delta^5 [4][E, F], their row sums P [4][N, F]) of mom_sum / mom_central (+ the chunk merges)"""
    S, _ = g.row_sums(m)
    mu = div(S, np.maximum(g.deg, 1))
    delta = m - mu[g.row]
    q = [delta * delta]
    for _ in range(3):
        q.append(q[-1] * delta)
    return mu, delta, q, [g.row_sums(v)[0] for v in q]


def moment_root(M, k, dm: DevMath):
    """sign(M) * powf(fl(|M| + 1e-5), fl(1/k)); 0 and NaN pass through"""
    live = (M > 0) | (M < 0)
    r = M.copy()
    if live.any():
        p = dm.powf(np.abs(M[live]) + EPS, INV_K[k])
        r[live] = np.where(M[live] > 0, p, -p)
    return r


def moment_slope(M, k, dm: DevMath):
    """fl(inv_k * powf(fl(|M| + 1e-5), e_k)); 0 where M == 0, NaN passes through"""
    live = (M > 0) | (M < 0)
    r = np.where(M == 0, F32(0), M).astype(F32)
    if live.any():
        r[live] = INV_K[k] * dm.powf(np.abs(M[live]) + EPS, SLOPE_E[k])
    return r


def weighted_rows(g: Graph, m, name, dm: DevMath):
    """y [N, F] of one weighted aggregator (rows without in-edges: 0) and the per-slot quantities the backward reuses"""
    if name == "normalised_mean":
        r = rsqrt_deg(g.deg)
        node = g.degree_node()
        rj = np.where((node >= 0) & (node < g.n), r[np.clip(node, 0, g.n - 1)], F32(0)).astype(F32)
        w = (r[g.row] * rj).astype(F32)
        y, _ = g.row_sums(m * w[:, None])
        return np.where((g.deg > 0)[:, None], y, F32(0)), {"w": w, "r": r, "rj": rj}
    sigma = F32(-1.0 if name == "softmin" else 1.0)
    n = sigma * m
    M = g.row_max(n)
    e = dm.expf(n - M[g.row])
    Z, _ = g.row_sums(e)
    S, _ = g.row_sums(e * n)
    with np.errstate(invalid="ignore", divide="ignore"):
        yp = S / Z
    y = np.where((g.deg > 0)[:, None], sigma * yp, F32(0))
    return y, {"n": n, "M": M, "e": e, "Z": Z, "S": S, "yp": yp}


# ---- output layout ------------------------------------------------------------------------------------------------------
def layout(F, towers, has_self, A, S):
    """(Ft, Wt, base [F]): the output column of feature f for (scaler 0, position 0) is base[f] (mom_base_col)"""
    Ft = F // towers
    Wt = (int(has_self) + A * S) * Ft
    f = np.arange(F)
    return Ft, Wt, (f // Ft) * Wt + int(has_self) * Ft + f % Ft


def code_of(name):
    if name in MOMENTS:
        return 6 + MOMENTS[name] - 3
    if name in WEIGHTED:
        return 9 + WEIGHTED.index(name)
    return None


# ---- forward ------------------------------------------------------------------------------------------------------------
def forward(g: Graph, x, bias, aggrs, scales, dm: DevMath, *, towers=1, has_self=False, flags=0, ldeg=None, out=None):
    """[N, T*Wt] with the add-on columns of every row the add-on kernels select written, everything else left as `out`
    (NaN by default).  Selection: light rows unless PNA_FLAG_SKIP_LIGHT (and, with a masked view, only rows whose
    light_deg >= 0), split rows unless PNA_FLAG_SKIP_HUBS."""
    N, F = g.n, x.shape[1]
    S, A = scales.shape[1], len(aggrs)
    Ft, Wt, base = layout(F, towers, has_self, A, S)
    if out is None:
        out = np.full((N, towers * Wt), np.nan, F32)
    sel = np.zeros(N, bool)
    if not flags & FLAG_SKIP_LIGHT:
        sel |= ~g.hub & (True if ldeg is None else np.asarray(ldeg) >= 0)
    if not flags & FLAG_SKIP_HUBS:
        sel |= g.hub
    m = g.messages(x, bias)
    zero_all = ((g.deg == 0) & bool(flags & FLAG_ZERO_ISOLATED))[:, None]
    vals = {}
    if any(a in MOMENTS for a in aggrs):
        _, _, _, P = central(g, m)
        for k in (3, 4, 5):
            M = div(P[k - 2], np.maximum(g.deg, 1))
            vals[f"moment{k}"] = np.where((g.deg > 0)[:, None], moment_root(M, k, dm), F32(0))
    for name in WEIGHTED:
        if name in aggrs:
            vals[name] = weighted_rows(g, m, name, dm)[0]
    rows = np.nonzero(sel)[0]
    for a, name in enumerate(aggrs):
        if name not in vals:
            continue
        y = vals[name][rows]
        for s in range(S):
            v = y * scales[rows, s:s + 1]          # the identity scaler's factor is 1: the skipped multiply is exact
            v = np.where(zero_all[rows], F32(0), v)
            out[rows[:, None], (base + (s * A + a) * Ft)[None, :]] = v
    return out


# ---- backward -----------------------------------------------------------------------------------------------------------
def upstream(go, base, aggrs, scales, name, Ft):
    """G [N, F]: the upstream gradient of `name`'s value summed over its list positions, then over the scalers, in order"""
    A, S = len(aggrs), scales.shape[1]
    G = np.zeros((go.shape[0], len(base)), F32)
    for a, nm in enumerate(aggrs):
        if nm != name:
            continue
        for s in range(S):
            v = go[:, base + (s * A + a) * Ft]
            G = G + scales[:, s:s + 1] * v
    return G


def moment_terms(g: Graph, m, go, aggrs, scales, base, Ft, dm: DevMath):
    """[E, F] per-slot moment term (0 in rows without in-edges), and the coefficients (a3, a4, a5, c0)"""
    orders = [k for k in (3, 4, 5) if f"moment{k}" in aggrs]
    mu, delta, q, P = central(g, m)
    d = np.maximum(g.deg, 1)
    G = {k: upstream(go, base, aggrs, scales, f"moment{k}", Ft) for k in (3, 4, 5)}
    kd = {k: div(np.full((g.n, 1), k, F32), d)[:, :1] for k in (3, 4, 5)}       # SharedDivisor of (float)k: fl(k / d)
    a, C = {}, {}
    for k in (3, 4, 5):
        C[k] = div(P[k - 3], d)                                                 # C_(k-1)
        a[k] = (G[k] * moment_slope(div(P[k - 2], d), k, dm)) * kd[k] if k in orders else np.zeros_like(C[k])
    c0 = np.zeros_like(C[3])
    for k in orders:
        c0 = c0 + a[k] * C[k]
    t = np.zeros_like(m)
    for k in orders:
        t = t + a[k][g.row] * q[k - 3]
    t = t - c0[g.row]
    return t, (a[3], a[4], a[5], c0)


def weighted_terms(g: Graph, m, go, aggrs, scales, base, Ft, name, dm: DevMath):
    """[E, F] per-slot term of one weighted aggregator (rows without in-edges emit nothing)"""
    G = upstream(go, base, aggrs, scales, name, Ft)
    _, p = weighted_rows(g, m, name, dm)
    if name == "normalised_mean":
        return G[g.row] * (p["r"][g.row] * p["rj"]).astype(F32)[:, None]
    with np.errstate(invalid="ignore", divide="ignore"):
        a, yp = G / p["Z"], p["yp"]
    return (a[g.row] * p["e"]) * (F32(1) + (p["n"] - yp[g.row]))


def addon_terms(g: Graph, x, bias, go, aggrs, scales, dm: DevMath, *, towers=1, has_self=False):
    """[(family, [E, F] term)] in launch order: moments, softmax, softmin, normalised_mean (those in the list)"""
    F = x.shape[1]
    Ft, _, base = layout(F, towers, has_self, len(aggrs), scales.shape[1])
    m = g.messages(x, bias)
    out = []
    if any(a in MOMENTS for a in aggrs):
        out.append(("moments", moment_terms(g, m, go, aggrs, scales, base, Ft, dm)[0]))
    for name in WEIGHTED:
        if name in aggrs:
            out.append((name, weighted_terms(g, m, go, aggrs, scales, base, Ft, name, dm)))
    return out


def core(g: Graph, x, bias, go, aggrs, scales, *, towers=1, has_self=False, relu_var=False):
    """backward_paths_ref's core term with the add-on codes as PNA_AGGR_SKIP: (gm [E, F], gb [N, F], chunk shares [C, F])"""
    stripped = ["_skip" if code_of(a) is not None else a for a in aggrs]
    st = B.row_stats_bwd(x, g.rowptr, g.col, g.hub_info, g.chunk, bias)
    c = B.coefficients(st, g.deg, go, np.asarray(scales), stripped, towers=towers, has_self=has_self, relu_var=relu_var)
    return B.slot_grads(c, st, x, g.rowptr, g.col, g.hub_info, g.chunk, bias)


def backward(g: Graph, x, bias, go, aggrs, scales, dm: DevMath, *, towers=1, has_self=False, relu_var=False):
    """What the per-slot instance (pna_aggregate_bwd_slots over all F columns; a slab is a column slice of it) and the
    atomic instance with col == None produce: (grad per slot [E, F], grad_row_bias [N, F], terms).  `terms` lists the core's
    term and every family's, [(name, [E, F])], for the order-free bound of the atomic instance with col."""
    gm, gb, _ = core(g, x, bias, go, aggrs, scales, towers=towers, has_self=has_self, relu_var=relu_var)
    terms = [("core", gm)]
    gs = gm.copy()
    gb = gb.copy()
    for name, t in addon_terms(g, x, bias, go, aggrs, scales, dm, towers=towers, has_self=has_self):
        gs = gs + t
        rs, _ = g.row_sums(t)
        live = g.deg > 0
        gb[live] = gb[live] + rs[live]
        terms.append((name, t))
    return gs, gb, terms


# ---- which kernels run ----------------------------------------------------------------------------------------------------
def addon_launches(aggrs, width, n_rows, n_hubs, n_chunks, *, backward=False, flags=0, row_bias_grad=True):
    """[(kernel, (gridDim.x, gridDim.y))] in launch order (launch_addons_fwd / launch_addons_bwd): gridDim.y =
    ceil(width / 32) with width = n_feat (forward, atomic backward) or f_count (per-slot backward), 8 rows or chunks per
    CTA.  Forward: SKIP_LIGHT drops the rows kernel, SKIP_HUBS the split-row chain; normalised_mean has no max pass; the
    backward's normalised_mean has no chunk pass at all, and k_mom_bwd_hub_bias runs only with grad_row_bias."""
    per = MOM_THREADS // 32
    gy = -(-width // 32)
    gx, gc, gh = -(-n_rows // per), -(-n_chunks // per), -(-n_hubs // per)
    W = 6 if backward else 4
    rows_k = not backward and bool(flags & FLAG_SKIP_LIGHT)
    hubs = n_hubs > 0 and (backward or not flags & FLAG_SKIP_HUBS)
    out = []
    if any(a in MOMENTS for a in aggrs):
        if not rows_k:
            out.append(("k_mom_bwd_rows" if backward else "k_mom_rows", (gx, gy)))
        if hubs:
            out += [(f"k_mom_chunk_sum<{W}>", (gc, gy)), (f"k_mom_hub_mean<{W}>", (gh, gy)),
                    (f"k_mom_chunk_central<{W}>", (gc, gy))]
            if backward:
                out += [("k_mom_bwd_hub_coef", (gh, gy)), ("k_mom_bwd_chunk_grad", (gc, gy))]
                if row_bias_grad:
                    out.append(("k_mom_bwd_hub_bias<6>", (gh, gy)))
            else:
                out.append(("k_mom_hub_final", (gh, gy)))
    for name in WEIGHTED:
        if name not in aggrs:
            continue
        nm = name == "normalised_mean"
        if not rows_k:
            out.append((f"k_wsum_bwd_rows[{name}]" if backward else f"k_wsum_rows[{name}]", (gx, gy)))
        if not hubs:
            continue
        if not nm:
            out += [(f"k_wsum_chunk_max<{W}>[{name}]", (gc, gy)), (f"k_wsum_hub_max<{W}>", (gh, gy))]
        if backward:
            if not nm:
                out.append((f"k_wsum_chunk_zs<6>[{name}]", (gc, gy)))
            out += [(f"k_wsum_bwd_hub_coef[{name}]", (gh, gy)), (f"k_wsum_bwd_chunk_grad[{name}]", (gc, gy))]
            if row_bias_grad:
                out.append(("k_mom_bwd_hub_bias<6>", (gh, gy)))
        else:
            out += [(f"k_wsum_chunk_zs<4>[{name}]", (gc, gy)), (f"k_wsum_hub_final[{name}]", (gh, gy))]
    return out
