"""fp32 restatements of pna_aggregate_fwd for the paths its launcher selects from the data -- TEST INFRASTRUCTURE (CPU only).

Rows below the split threshold are reduced slot by slot in CSR order (sum += m; sq += fl32(m*m); min; max), exactly as the
plain-C oracle (oracle/c/pna_oracle.c) does; tests/test_forward_paths_host.py checks the two agree bit for bit.  Split rows
are restated in the order the kernels merge their chunk partials (pna_b200/csrc/pna_aggregate_impl.cuh):
  * chunk partials: the same slot-by-slot reduction over `chunk_edges` consecutive slots of the row;
  * "sequential": the partials in chunk order (k_hub_finalize with <= 8 chunks);
  * "two_level": group q merges chunks q, q+8, .. in order, then groups 0..7 in order (k_hub_finalize, fold_split_row);
  * "tree": the radix-32 walk of k_hub_tree over the global chunk array, for every split row of the graph, when the
    largest in-degree exceeds 512 * chunk_edges and the lane group is a full warp.
The epilogue is the C oracle's, in float32: IEEE division by the in-degree, var = msq - mean*mean,
std = sqrt(relu(var) + 1e-5), one fp32 multiply per scaler.  A float64 evaluation of the same formulas (stats_f64) only
sanity-checks the restatement.  numpy float32 arithmetic rounds every operation and never contracts a multiply-add.
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
FIN_GROUPS = 8          # kFinGroups
TREE_R = 32             # kTreeR
TREE_MIN_CHUNKS = 512   # pna_aggregate_fwd: hub_merged when max_degree > 512 * chunk_edges
AGGR = ("sum", "mean", "min", "max", "var", "std")


# ---- which kernel instance the launcher picks (launch_typed / launch_config) ------------------------------------------
def lane_group(n_feat: int, elem_bytes: int, vec_ok: bool) -> tuple:
    """(G, K, feature blocks) of launch_typed for a row of n_feat elements."""
    vec = 16 // elem_bytes if vec_ok else 1
    chunks = n_feat // vec
    for lim, g in ((1, 1), (2, 2), (4, 4), (8, 8), (16, 16), (32, 32)):
        if chunks <= lim:
            return g, 1, 1
    k = 2 if chunks <= 64 else (3 if chunks <= 96 else 4)
    return 32, k, -(-n_feat // (32 * vec * k))


def merge_kind(max_degree: int, chunk_edges: int, group: int) -> str:
    """How the split rows' partials are merged: the radix tree needs a full warp per row (G == 32)."""
    return "tree" if (max_degree > TREE_MIN_CHUNKS * chunk_edges and group == 32) else "two_level"


# ---- graphs of the GPU tests (CPU-generated, seeded) ----------------------------------------------------------------------
def _with_rows(rng, n, n_random, lo, fixed):
    """n_random random edges into rows >= lo, plus fixed[r] in-edges into row r; sources uniform over the n rows."""
    dst = [rng.integers(lo, n, n_random)] + [np.full(d, r) for r, d in fixed.items()]
    dst = np.concatenate(dst)
    src = rng.integers(0, n, dst.size)
    p = rng.permutation(dst.size)
    return src[p], dst[p]


def split_graph(name: str):
    """(src, dst, n, split_threshold, chunk_edges) of the split-row graphs:
    tree3   -- a 3302-edge row (1101 chunks of 3: > 32^2, three tree levels) beside 40 split rows of 6..97 chunks;
    edge512 -- largest row exactly 512 * chunk_edges (two-level merge); edge513 -- one edge more (radix tree);
    wide128 -- the default-sized chunk: a 520-chunk row (> 512 * 128 in-edges) and 9 split rows of 2..10 chunks."""
    rng = np.random.default_rng(sum(map(ord, name)))
    if name == "tree3":
        fixed = {0: 3 * 1100 + 2, **{r: 16 + 7 * r for r in range(1, 41)}}
        return (*_with_rows(rng, 600, 3000, 41, fixed), 600, 16, 3)
    if name in ("edge512", "edge513"):
        fixed = {0: int(name[4:]), **{r: 8 + 5 * r for r in range(1, 20)}}
        return (*_with_rows(rng, 300, 1200, 20, fixed), 300, 8, 1)
    if name == "wide128":
        fixed = {0: 128 * 520 + 1, **{r: 128 * r + 7 for r in range(1, 10)}}
        return (*_with_rows(rng, 2000, 10000, 10, fixed), 2000, 128, 128)
    raise KeyError(name)


def tail_graph(n: int = 150_000, seed: int = 5):
    """(src, dst, n): 0..8 in-edges per row and 16 rows of 300..3000 (split rows at the default threshold of 256)."""
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 9, n)
    deg[rng.choice(n, 16, replace=False)] = rng.integers(300, 3000, 16)
    dst = np.repeat(np.arange(n), deg)
    src = rng.integers(0, n, dst.size)
    p = rng.permutation(dst.size)
    return src[p], dst[p], n


# ---- host CSR (the layout build_csr produces; hub order is a parameter, the GPU hands hubs out in atomic order) ---------
def host_csr(src, dst, n: int, split: int, chunk: int, hub_order=None):
    """rowptr, col (stable sort by destination), hub_info [H, 4] = (row, first chunk, n chunks, degree), chunk_items [C, 2]."""
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    order = np.argsort(dst, kind="stable")
    col = src[order]
    deg = np.bincount(dst, minlength=n)
    rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    hubs = np.nonzero(deg >= split)[0]
    if hub_order is not None:
        hubs = hubs[np.asarray(hub_order)]
    info, items, first = [], [], 0
    for h, r in enumerate(hubs):
        nch = -(-int(deg[r]) // chunk)
        info.append((r, first, nch, deg[r]))
        items += [(h, j) for j in range(nch)]
        first += nch
    return rowptr, col, np.array(info, np.int64).reshape(-1, 4), np.array(items, np.int64).reshape(-1, 2)


# ---- reductions --------------------------------------------------------------------------------------------------------
def segment_stats(x, col, beg, length, bias=None, bias_rows=None):
    """[R, 4, F] float32 (sum, sumsq, min, max) of R slot segments [beg, beg + length), slot by slot in slot order.
    With bias, every message is fl32(x[src] + bias[bias_rows[r]]) (the kernel adds the row bias before anything else)."""
    R, F = len(beg), x.shape[1]
    st = np.empty((R, 4, F), F32)
    st[:, 0] = 0
    st[:, 1] = 0
    st[:, 2] = np.inf
    st[:, 3] = -np.inf
    beg, length = np.asarray(beg, np.int64), np.asarray(length, np.int64)
    for k in range(int(length.max()) if R else 0):
        act = np.nonzero(length > k)[0]
        m = x[col[beg[act] + k]]
        if bias is not None:
            m = m + bias[bias_rows[act]]
        st[act, 0] = st[act, 0] + m
        st[act, 1] = st[act, 1] + m * m
        st[act, 2] = np.minimum(st[act, 2], m)
        st[act, 3] = np.maximum(st[act, 3], m)
    return st


def _acc(F):
    a = np.empty((4, F), F32)
    a[0] = a[1] = 0
    a[2], a[3] = np.inf, -np.inf
    return a


def add_into(acc, p):
    """One merge step of merge_partials / k_hub_tree: fp32 adds of sum and sumsq, min, max."""
    acc[0] = acc[0] + p[0]
    acc[1] = acc[1] + p[1]
    acc[2] = np.minimum(acc[2], p[2])
    acc[3] = np.maximum(acc[3], p[3])


def merge_sequential(P, first, nch):
    acc = _acc(P.shape[2])
    for c in range(first, first + nch):
        add_into(acc, P[c])
    return acc


def merge_two_level(P, first, nch):
    if nch <= FIN_GROUPS:
        return merge_sequential(P, first, nch)
    groups = []
    for q in range(FIN_GROUPS):
        g = _acc(P.shape[2])
        for c in range(first + q, first + nch, FIN_GROUPS):
            add_into(g, P[c])
        groups.append(g)
    acc = _acc(P.shape[2])
    for g in groups:
        add_into(acc, g)
    return acc


def tree_walk(n_chunks, first_of_chunk):
    """The additions of k_hub_tree, in order: (S, head, pos) = P[head] += P[pos] at the level with stride S."""
    steps, S = [], 1
    while S < n_chunks:
        for base in range(0, n_chunks, TREE_R * S):
            for j in range(1, TREE_R):
                pos = base + j * S
                if pos >= n_chunks:
                    break
                first = int(first_of_chunk[pos])
                if first < pos:
                    steps.append((S, max(first, base), pos))
        S *= TREE_R
    return steps


def merge_tree(P, hub_info, chunk_items):
    """k_hub_tree over a copy of the global partial array; returns [H, 4, F]: every split row's total (its first slot)."""
    P = P.copy()
    first_of_chunk = hub_info[chunk_items[:, 0], 1] if len(chunk_items) else np.zeros(0, np.int64)
    for _, head, pos in tree_walk(len(P), first_of_chunk):
        add_into(P[head], P[pos])
    return P[hub_info[:, 1]] if len(hub_info) else np.zeros((0,) + P.shape[1:], F32)


def chunk_partials(x, rowptr, col, hub_info, chunk_items, chunk_edges, bias=None):
    """[C, 4, F] float32 partial of every chunk of every split row (k_hub_chunks / the streamed kernel's pseudo-rows)."""
    h, j = chunk_items[:, 0], chunk_items[:, 1]
    row, deg = hub_info[h, 0], hub_info[h, 3]
    beg = rowptr[row] + j * chunk_edges
    length = np.minimum(chunk_edges, deg - j * chunk_edges)
    return segment_stats(x, col, beg, length, bias, row)


def row_stats(x, rowptr, col, hub_info, chunk_items, chunk_edges, merge, bias=None):
    """[N, 4, F] float32 statistics of every destination row as the kernels compute them."""
    N = len(rowptr) - 1
    deg = np.diff(rowptr)
    st = segment_stats(x, col, rowptr[:-1], np.where(np.isin(np.arange(N), hub_info[:, 0]), 0, deg), bias, np.arange(N))
    if len(hub_info):
        P = chunk_partials(x, rowptr, col, hub_info, chunk_items, chunk_edges, bias)
        if merge == "tree":
            st[hub_info[:, 0]] = merge_tree(P, hub_info, chunk_items)
        else:
            fn = merge_two_level if merge == "two_level" else merge_sequential
            for r, first, nch, _ in hub_info:
                st[r] = fn(P, first, nch)
    return st


def stats_f64(x, rowptr, col, bias=None):
    """float64 (sum, sumsq, min, max) per row: the same formulas, no fp32 rounding."""
    N = len(rowptr) - 1
    dst = np.repeat(np.arange(N), np.diff(rowptr))
    m = x[col].astype(np.float64)
    if bias is not None:
        m = m + bias[dst].astype(np.float64)
    st = np.zeros((N, 4, x.shape[1]), np.float64)
    np.add.at(st[:, 0], dst, m)
    np.add.at(st[:, 1], dst, m * m)
    st[:, 2], st[:, 3] = np.inf, -np.inf
    np.minimum.at(st[:, 2], dst, m)
    np.maximum.at(st[:, 3], dst, m)
    return st


# ---- epilogue -----------------------------------------------------------------------------------------------------------
def host_scales(deg, scalers, avg_log, avg_lin):
    """[N, S] factors of the scalers that need no logarithm (identity, linear, inverse_linear) in float32."""
    d = np.asarray(deg).astype(F32)
    iso = d == 0
    cols = []
    for s in scalers:
        if s == "identity":
            cols.append(np.ones_like(d))
        elif s == "linear":
            cols.append(d / F32(avg_lin))
        elif s == "inverse_linear":
            cols.append(np.where(iso, F32(1), F32(avg_lin) / np.where(iso, F32(1), d)))
        else:
            raise ValueError(f"{s}: take the factors from pna_b200.aggregate.row_scales")
    return np.stack(cols, 1).astype(F32)


def epilogue(st, deg, aggrs, scales, *, towers=1, self_feat=None, self_divided=True, zero_isolated=False, relu_var=False):
    """[N, towers * (has_self + S*A) * Ft] in the kernel's column order from per-row statistics (float32 or float64)."""
    dt = st.dtype.type
    N, _, F = st.shape
    deg = np.asarray(deg)
    iso = (deg == 0)[:, None]
    cnt = np.maximum(deg, 1).astype(dt)[:, None]
    mean = st[:, 0] / cnt
    var = st[:, 1] / cnt - mean * mean
    vals = {"sum": st[:, 0], "mean": mean, "min": np.where(iso, dt(0), st[:, 2]), "max": np.where(iso, dt(0), st[:, 3]),
            "var": np.maximum(var, dt(0)) if relu_var else var, "std": np.sqrt(np.maximum(var, dt(0)) + dt(1e-5))}
    scales = np.asarray(scales).astype(dt)
    T, A, S = towers, len(aggrs), scales.shape[1]
    Ft = F // T
    hs = self_feat is not None
    Wt = (int(hs) + A * S) * Ft
    out = np.empty((N, T * Wt), dt)
    for t in range(T):
        o = t * Wt
        if hs:
            out[:, o:o + Ft] = self_feat[:, t * Ft:(t + 1) * Ft] if self_divided else self_feat[:, :Ft]
            o += Ft
        for s in range(S):
            for a, name in enumerate(aggrs):
                v = vals[name][:, t * Ft:(t + 1) * Ft]
                v = v * scales[:, s:s + 1]
                if zero_isolated:
                    v = np.where(iso, dt(0), v)
                out[:, o + (s * A + a) * Ft:o + (s * A + a + 1) * Ft] = v
    return out
