"""numpy restatement of the tensor-core linear (pna_b200/csrc/pna_linear.cu) -- TEST INFRASTRUCTURE (CPU only).

Every operand x goes through `split`: hi = tf32_rna(x) (cvt.rna.satfinite.tf32.f32), lo = tf32_rna(fl32(x - hi))
(cvt.rna.tf32.f32).  An output is two tensor-core accumulation chains, acc = sum hi.hi and corr = sum (hi.lo + lo.hi) (the
lo.lo product is never formed), then fp32 round-to-nearest adds in the order the kernels issue them:
  * k_linear_3xtf32 (forward, and the data gradient): y = fl(fl(acc + corr) + b), b = +0.0 without a bias.  Pipeline steps
    run compact-block-major, scaler-minor; the loaders split fl32(c_s(i) * a).  With FOLD (the data gradient when
    n_out * S / 32 > kLinFoldSteps) the chains restart every kLinFoldSteps steps, never after the last one, and
    Y <- fl(Y + fl(fl(acc_g + corr_g) + 0)).  The data gradient runs on fl32(c_s * dY) with the re-blocked weight
    W''[c, s * O + o] = W[o, s * n_cols + c], in column slabs.
  * k_linear_bwd_weight: per split of the rows, part <- fl(part + fl(acc + corr)) every kWgFoldRows rows and after the
    last K block; k_sum_splits then adds the partials in ascending split order (one split: dW is the partial).
The chain sums are an input of the restatement: `chains` forms them in float64.  On grid data (`grid_*`: terms that are
multiples of one power of two u with sum |terms| <= 2^12 u) float64 sums them exactly and so does the tensor core, in any
order; on random data the exactly summed restatement R gives an elementwise bar (`bar_*`).
The keyword arguments of the restatements select the alternatives the tests must be able to tell apart (other fold
periods, descending split order, lo.lo included, a truncating split, scaling after the split, the unsaturated split).
"""
from __future__ import annotations

import numpy as np

F32 = np.float32
LIN_BK = 32                 # kLinBK: fp32 per K block
LIN_FOLD_STEPS = 4          # kLinFoldSteps
WG_FOLD_ROWS = 64           # kWgFoldRows
WG_MIN_SPLIT_ROWS = 512     # kWgMinSplitRows
WG_TARGET_CTAS = 264        # kWgTargetCtas
TF32_MAX_BITS = 0x7F7FE000  # the largest finite TF32 value: what satfinite clamps to


# ---- the TF32 split ------------------------------------------------------------------------------------------------
def tf32_rna(x, satfinite: bool = False):
    """cvt.rna[.satfinite].tf32.f32 on fp32 bits: finite x -> (bits + 0x1000) & 0xffffe000 (ties away from zero), inf and
    NaN -> bits & 0xffffe000.  satfinite: a result that became inf (|x| >= 0x7F7FF000) and an inf input give +-MAX."""
    x = np.asarray(x, dtype=F32)
    b = x.view(np.uint32).astype(np.uint64)
    mag = b & 0x7FFFFFFF
    finite = mag < 0x7F800000
    r = np.where(finite, (b + 0x1000) & 0xFFFFE000, b & 0xFFFFE000)
    if satfinite:
        rmag = r & 0x7FFFFFFF
        r = np.where(rmag == 0x7F800000, (r & 0x80000000) | TF32_MAX_BITS, r)
    return r.astype(np.uint32).view(F32).reshape(x.shape)


def tf32_rz(x):
    """cvt.rz.tf32.f32: the truncating split the kernel must not use (an alternative)."""
    x = np.asarray(x, dtype=F32)
    return (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(F32).reshape(x.shape)


def split(x, mode: str = "rna"):
    """(hi, lo) of the loaders and k_split_weight[_t]: mode "rna" (the kernel), "rna_unsat" (hi without satfinite: the
    split before FLT_MAX was handled), "rz" (truncating)."""
    x = np.asarray(x, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        if mode == "rz":
            hi = tf32_rz(x)
            return hi, tf32_rz(x - hi)
        hi = tf32_rna(x, satfinite=(mode == "rna"))
        return hi, tf32_rna(x - hi)


# ---- launch choices (pure functions of the shape) ---------------------------------------------------------------------
def lin_rows(o: int) -> int:
    return 128 if o <= 128 else 64


def lin_stages(o: int) -> int:
    return 3 if o <= 128 else 2


def k_ahead(o: int) -> int:
    """kAhead = 8 / kSlabs: K blocks of A in flight per loader thread."""
    return 8 // (lin_rows(o) // 32)


def bwd_data_slab(n_cols: int) -> int:
    return 64 if (n_cols + 63) // 64 * 64 < (n_cols + 127) // 128 * 128 else 128


def bwd_data_slabs(n_cols: int):
    """(slab width, slab count, width of the last slab)."""
    os_ = bwd_data_slab(n_cols)
    n = -(-n_cols // os_)
    return os_, n, n_cols - (n - 1) * os_


def bwd_data_fold(n_out: int, n_rep: int) -> bool:
    """pna_linear_bwd_data launches the FOLD instance when n_out * S / 32 > kLinFoldSteps."""
    return n_out * n_rep // LIN_BK > LIN_FOLD_STEPS


def bwd_weight_plan(n_rows: int, n_in: int, n_out: int):
    """(col_tiles, o_tiles, n_split, rows per split) of pna_linear_bwd_weight."""
    col_tiles = -(-n_in // 128)
    o_tiles = 2 if n_out > 128 else 1
    tiles = col_tiles * o_tiles
    sp = min(-(-n_rows // WG_MIN_SPLIT_ROWS), max(1, -(-WG_TARGET_CTAS // tiles)))
    sp = max(sp, 1)
    rows = (-(-n_rows // sp) + 31) // 32 * 32
    return col_tiles, o_tiles, -(-n_rows // rows), rows


def fwd_workspace_bytes(n_in: int, n_out: int) -> int:
    return 2 * n_in * n_out * 4


def bwd_workspace_bytes(n_rows: int, n_in: int, n_out: int, n_rep: int) -> int:
    n_cols = n_in // n_rep
    os_ = bwd_data_slab(n_cols)
    data = 2 * n_out * n_rep * (-(-n_cols // os_) * os_) * 4
    weight = 0
    if n_rows > 0:
        _, _, n_split, _ = bwd_weight_plan(n_rows, n_in, n_out)
        weight = n_split * n_out * n_in * 4 if n_split > 1 else 0
    return max(data, weight)


# ---- operands in pipeline-step order ---------------------------------------------------------------------------------
def scaled_steps(a, c):
    """[N, n_it * 32]: the loaders' operand fl32(c_s(i) * a) in pipeline-step order (compact block kb, scaler s) ->
    step kb * S + s.  c None: a itself."""
    a = np.asarray(a, dtype=F32)
    if c is None:
        return a
    n, k = a.shape
    s_n = c.shape[1]
    with np.errstate(invalid="ignore", over="ignore"):
        blocks = np.stack([a * c[:, s:s + 1].astype(F32) for s in range(s_n)], axis=1)       # [N, S, K]
    return blocks.reshape(n, s_n, k // LIN_BK, LIN_BK).transpose(0, 2, 1, 3).reshape(n, -1)


def weight_steps(w, n_rep: int):
    """[O, n_it * 32]: the weight's K blocks in pipeline-step order (step kb * S + s reads block s * n_kb + kb)."""
    w = np.asarray(w, dtype=F32)
    o, k = w.shape
    n_kb = k // n_rep // LIN_BK
    return w.reshape(o, n_rep, n_kb, LIN_BK).transpose(0, 2, 1, 3).reshape(o, -1)


def reblock_weight(w, n_rep: int):
    """W''[c, s * O + o] = W[o, s * n_cols + c]: the data gradient's weight, [n_cols, S * O]."""
    o, n_in = w.shape
    n_cols = n_in // n_rep
    return np.asarray(w, dtype=F32).reshape(o, n_rep, n_cols).transpose(2, 1, 0).reshape(n_cols, n_rep * o)


def _split_operand(x, c, mode, scale_after):
    """(hi, lo) of the scaled operand in step order; scale_after: split a, then scale the parts (an alternative)."""
    if c is None or not scale_after:
        return split(scaled_steps(x, c), mode)
    hi, lo = split(np.asarray(x, dtype=F32), mode)
    return scaled_steps(hi, c), scaled_steps(lo, c)


# ---- chains -----------------------------------------------------------------------------------------------------------
def chains(xh, xl, wh, wl, k0: int, k1: int, lolo: bool = False):
    """float64 (acc, corr, sum |acc terms|, sum |corr terms|) of the K range [k0, k1): xh/xl [M, K], wh/wl [N, K]."""
    xh, xl = xh[:, k0:k1].astype(np.float64), xl[:, k0:k1].astype(np.float64)
    wh, wl = wh[:, k0:k1].astype(np.float64), wl[:, k0:k1].astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        acc = xh @ wh.T
        corr = xh @ wl.T + xl @ wh.T
        if lolo:
            corr = corr + xl @ wl.T
        s_acc = np.abs(xh) @ np.abs(wh).T
        s_corr = np.abs(xh) @ np.abs(wl).T + np.abs(xl) @ np.abs(wh).T
    return acc, corr, s_acc, s_corr


def _f32(x):
    with np.errstate(invalid="ignore", over="ignore"):
        return np.asarray(x).astype(F32)


def _groups(n_steps: int, fold):
    """K-block ranges of the accumulation chains: one chain, or a restart every `fold` steps (never after the last)."""
    if not fold:
        return [(0, n_steps)]
    return [(g, min(g + fold, n_steps)) for g in range(0, n_steps, fold)]


def linear_restate(xh, xl, wh, wl, bias=None, fold=None, lolo=False, bars=False):
    """k_linear_3xtf32 on split operands in step order ([M, n_it*32], [N, n_it*32]) -> fp32 [M, N].  fold: steps per chain
    (None: one chain).  bars: also return the elementwise bar of the random tier (see `bar_from_chains`)."""
    n_steps = xh.shape[1] // LIN_BK
    y = None
    bar = np.zeros((xh.shape[0], wh.shape[0]))
    groups = _groups(n_steps, fold)
    zero = np.zeros(wh.shape[0], dtype=F32)
    for gi, (g0, g1) in enumerate(groups):
        acc, corr, s_acc, s_corr = chains(xh, xl, wh, wl, g0 * LIN_BK, g1 * LIN_BK, lolo)
        b = bias.astype(F32) if (bias is not None and gi == len(groups) - 1) else zero
        with np.errstate(invalid="ignore", over="ignore"):
            v = (_f32(acc) + _f32(corr)) + b[None, :]
            y = v if y is None else y + v
        bar += bar_from_chains(s_acc, s_corr, g1 - g0)
    return (y, bar) if bars else y


def bar_from_chains(s_acc, s_corr, n_blocks):
    """(m + 1) 2^-23 sum|terms| per chain, m = k8 MMAs into the accumulator: 4 per K block for hi.hi, 8 for the cross
    terms (one truncation per MMA keeping at least 24 bits)."""
    return (4 * n_blocks + 1) * 2.0 ** -23 * s_acc + (8 * n_blocks + 1) * 2.0 ** -23 * s_corr


def fwd_restate(a, w, bias=None, c=None, mode="rna", lolo=False, scale_after=False, bars=False):
    """pna_linear_fwd (c None) / pna_linear_scaled_fwd: a [N, K], w [O, S*K], c [N, S]."""
    n_rep = 1 if c is None else c.shape[1]
    xh, xl = _split_operand(a, c, mode, scale_after)
    wh, wl = split(weight_steps(w, n_rep), mode)
    return linear_restate(xh, xl, wh, wl, bias, None, lolo, bars)


def bwd_data_restate(gy, w, c=None, mode="rna", lolo=False, scale_after=False, fold="auto", bars=False):
    """pna_linear_bwd_data: grad_y [N, O], w [O, n_in], c [N, S] -> grad_a [N, n_in / S].  fold "auto": the launcher's
    choice (kLinFoldSteps, or no fold when n_out * S / 32 <= kLinFoldSteps)."""
    o = w.shape[0]
    n_rep = 1 if c is None else c.shape[1]
    if fold == "auto":
        fold = LIN_FOLD_STEPS if bwd_data_fold(o, n_rep) else None
    xh, xl = _split_operand(gy, c, mode, scale_after)
    wh, wl = split(reblock_weight(w, n_rep), mode)          # W'' [n_cols, S*O]: step t reads block t of W'' (below)
    # step kb * S + s of the kernel reads W'' block s * n_kb + kb, where n_kb = O / 32: the same re-ordering as the forward
    wh, wl = weight_steps(wh, n_rep), weight_steps(wl, n_rep)
    return linear_restate(xh, xl, wh, wl, None, fold, lolo, bars)


def bwd_weight_restate(gy, a, c=None, mode="rna", lolo=False, scale_after=False, fold_rows=WG_FOLD_ROWS,
                       order="asc", bars=False):
    """pna_linear_bwd_weight: grad_y [N, O], a [N, n_a], c [N, S] -> dW [O, S * n_a]."""
    n, o = gy.shape
    n_rep = 1 if c is None else c.shape[1]
    n_in = a.shape[1] * n_rep
    if c is None or not scale_after:
        ap = np.asarray(a, dtype=F32) if c is None else np.concatenate(
            [np.asarray(a, dtype=F32) * c[:, s:s + 1].astype(F32) for s in range(n_rep)], axis=1)
        with np.errstate(invalid="ignore", over="ignore"):
            ah, al = split(ap, mode)
    else:
        h, l = split(np.asarray(a, dtype=F32), mode)
        ah = np.concatenate([h * c[:, s:s + 1].astype(F32) for s in range(n_rep)], axis=1)
        al = np.concatenate([l * c[:, s:s + 1].astype(F32) for s in range(n_rep)], axis=1)
    yh, yl = split(np.asarray(gy, dtype=F32), mode)
    _, _, n_split, rows = bwd_weight_plan(n, n_in, o)
    parts, bar = [], np.zeros((o, n_in))
    for sp in range(n_split):
        r0, r1 = sp * rows, min(n, (sp + 1) * rows)
        part = None
        for g0 in range(r0, r1, fold_rows):
            g1 = min(g0 + fold_rows, r1)
            acc, corr, s_acc, s_corr = chains(yh.T, yl.T, ah.T, al.T, g0, g1, lolo)
            with np.errstate(invalid="ignore", over="ignore"):
                v = _f32(acc) + _f32(corr)
                part = v if part is None else part + v
            bar += bar_from_chains(s_acc, s_corr, -(-(g1 - g0) // LIN_BK))
        parts.append(part)
    seq = parts if order == "asc" else parts[::-1]
    dw = seq[0]
    with np.errstate(invalid="ignore", over="ignore"):
        for p in seq[1:]:
            dw = dw + p
    return (dw, bar) if bars else dw


def rounding_slack(r, n_adds):
    """fp32 roundings after the chains (the epilogue, the folds, the split sums): n_adds ulps of the result."""
    return n_adds * 2.0 ** -23 * np.abs(r.astype(np.float64))


# ---- grid data (the exact tier) --------------------------------------------------------------------------------------
def grid_matrix(rng, shape, e: int, density: float, lo_shift: int = 18, positive: float = 0.8):
    """hi = m 2^e (m in 1..3, positive with probability `positive`), lo = +-2^(e - lo_shift) on half the nonzeros.
    |lo| < half a TF32 ulp of hi and x = hi + lo is exact in fp32, so split(x) == (hi, lo)."""
    nz = rng.random(shape) < density
    m = rng.integers(1, 4, shape) * np.where(rng.random(shape) < positive, 1, -1)
    hi = (nz * m).astype(np.float64) * 2.0 ** e
    lo = nz * (rng.random(shape) < 0.5) * rng.choice([-1.0, 1.0], shape) * 2.0 ** (e - lo_shift)
    return hi.astype(F32), lo.astype(F32)


GRID_SCALES = (0.0, 0.5, 1.0, 1.5, 2.0, 3.0)   # dyadic factors with few bits, 0 (amplification of an isolated row) and 1


def grid_scales(rng, n: int, s_n: int):
    c = rng.choice(GRID_SCALES, (n, s_n)).astype(F32)
    c[:, 0] = 1.0
    return c


# probe values: x = 2^e - 2^(e-12) (negative lo: rna and truncation split it differently) against w = 2^ew + 2^(ew-12):
# the product's lo.lo term is one ulp of the result, so dropping it, or forming it from other parts, shows in the bits.
# The scale probe: x = 2^e + 3 * 2^(e-13) times c = 1.5 crosses half a TF32 ulp, so split(fl(c x)) != (c hi, c lo).
# Other rows are zero in the probes' K columns, which keeps every chain within the budget.
def probe_x(e):
    return F32(2.0 ** e - 2.0 ** (e - 12))


def probe_w(ew, sign=1.0):
    return F32(sign * (2.0 ** ew + 2.0 ** (ew - 12)))


def probe_scaled_x(e):
    return F32(2.0 ** e + 3 * 2.0 ** (e - 13))


PROBE_SCALE = 1.5


def grid_fwd(seed, n, k, o, s_n=0, bias=True, e=-3, ew=-4):
    """(a, w, bias, c) grid operands of pna_linear_fwd / _scaled_fwd.  Row 1 is the split probe, row 2 (scaled) the scale
    probe: c = (0, 1.5, 0, ..) and one nonzero at compact column 3."""
    rng = np.random.default_rng(seed)
    rep = max(s_n, 1)
    kt = rep * k
    dens = min(0.9, 180.0 / kt)
    ah, al = grid_matrix(rng, (n, k), e, dens)
    wh, wl = grid_matrix(rng, (o, kt), ew, 0.9, lo_shift=19)
    a, w = ah + al, wh + wl
    c = grid_scales(rng, n, s_n) if s_n else None
    kp = 5 % k
    a[:, kp] = 0
    if n > 1:
        a[1, :] = 0
        a[1, kp] = probe_x(e)
        if c is not None:
            c[1, :] = 1.0
    sg = rng.choice([-1.0, 1.0], o).astype(F32)
    for s in range(rep):
        w[:, s * k + kp] = probe_w(ew) * sg
    if c is not None and n > 2:
        kq = 3 % k if k > 3 else 0
        if kq == kp:
            kq = (kp + 1) % k
        a[:, kq] = 0
        a[2, :] = 0
        a[2, kq] = probe_scaled_x(e)
        c[2, :] = 0
        c[2, 1] = PROBE_SCALE
        for s in range(rep):
            w[:, s * k + kq] = probe_w(ew) * sg
    b = (rng.integers(-3, 4, o) * 2.0 ** (e + ew - 3)).astype(F32) if bias else None   # small: the probes' last bits show
    return a, w, b, c


def grid_bwd_data(seed, n, n_cols, o, s_n=0, e=-3, ew=-4):
    """(grad_y, w, c) grid operands of pna_linear_bwd_data.  The kernel's x is grad_y (K = O per scaler), its weight
    W''[c, s*O + o] = W[o, s*n_cols + c]: probe column o_p of grad_y is a row of W."""
    rng = np.random.default_rng(seed)
    rep = max(s_n, 1)
    kt = rep * o
    dens = min(0.9, 250.0 / min(kt, LIN_FOLD_STEPS * LIN_BK))
    yh, yl = grid_matrix(rng, (n, o), e, dens)
    wh, wl = grid_matrix(rng, (o, rep * n_cols), ew, 0.9, lo_shift=19)
    gy, w = yh + yl, wh + wl
    c = grid_scales(rng, n, s_n) if s_n else None
    op = 5 % o
    sg = rng.choice([-1.0, 1.0], n_cols).astype(F32)
    gy[:, op] = 0
    if n > 1:
        gy[1, :] = 0
        gy[1, op] = probe_x(e)
        if c is not None:
            c[1, :] = 1.0
    for s in range(rep):
        w[op, s * n_cols:(s + 1) * n_cols] = probe_w(ew) * sg
    if c is not None and n > 2:
        oq = 3
        gy[:, oq] = 0
        gy[2, :] = 0
        gy[2, oq] = probe_scaled_x(e)
        c[2, :] = 0
        c[2, 1] = PROBE_SCALE
        for s in range(rep):
            w[oq, s * n_cols:(s + 1) * n_cols] = probe_w(ew) * sg
    return gy, w, c


def grid_bwd_weight(seed, n, n_a, o, s_n=0, e=-3, ew=-4):
    """(grad_y, a, c) grid operands of pna_linear_bwd_weight.  The reduction runs over rows: the probes are crosses, row
    i_p of grad_y nonzero only in column o_p and column o_p nonzero only in row i_p, row i_p of a all probe_w.  Row 2 is
    the scale probe (a = probe_scaled_x, c = (0, 1.5, 0..), grad_y = probe_w in column 3 only)."""
    rng = np.random.default_rng(seed)
    rep = max(s_n, 1)
    yh, yl = grid_matrix(rng, (n, o), e, 0.7)
    ah, al = grid_matrix(rng, (n, n_a), ew, 0.7, lo_shift=19)
    gy, a = yh + yl, ah + al
    c = grid_scales(rng, n, s_n) if s_n else None
    if n > 1:
        gy[:, 1] = 0
        gy[1, :] = 0
        gy[1, 1] = probe_x(e)
        a[1, :] = probe_w(ew) * rng.choice([-1.0, 1.0], n_a).astype(F32)
        if c is not None:
            c[1, :] = 1.0
    if c is not None and n > 2 and o > 3:
        gy[:, 3] = 0
        gy[2, :] = 0
        gy[2, 3] = probe_w(e)
        a[2, :] = probe_scaled_x(ew) * rng.choice([-1.0, 1.0], n_a).astype(F32)
        c[2, :] = 0
        c[2, 1] = PROBE_SCALE
    return gy, a, c


# ---- budget: every chain's terms are multiples of one power of two u with sum |terms| <= 2^12 u ------------------------
def _low_exp(v):
    """Exponent of the lowest set bit of every (dyadic float64) entry; +inf for zeros."""
    v = np.abs(v)
    nz = v != 0
    _, ex = np.frexp(np.where(nz, v, 1.0))
    m = np.ldexp(np.where(nz, v, 1.0), 53 - ex).astype(np.int64)        # integer mantissas
    tz = np.log2((m & -m).astype(np.float64)).astype(np.int64)
    return np.where(nz, (ex - 53 + tz).astype(np.float64), np.inf)


def chain_budget(xh, xl, wh, wl, groups):
    """max over chains of sum|terms| / u, u the lowest bit any of the chain's terms has (terms of acc and of corr
    separately), for K-block ranges `groups`."""
    worst = 0.0
    for g0, g1 in groups:
        k0, k1 = g0 * LIN_BK, g1 * LIN_BK
        X = [xh[:, k0:k1].astype(np.float64), xl[:, k0:k1].astype(np.float64)]
        W = [wh[:, k0:k1].astype(np.float64), wl[:, k0:k1].astype(np.float64)]
        lx = [_low_exp(m) for m in X]
        lw = [_low_exp(m) for m in W]
        for pairs in (((0, 0),), ((0, 1), (1, 0))):
            s = sum(np.abs(X[i]) @ np.abs(W[j]).T for i, j in pairs)
            # the lowest bit of a product is the sum of its factors' lowest bits: min over k of lx[i, k] + lw[j, k]
            low = np.full(s.shape, np.inf)
            for i, j in pairs:
                for k in range(k1 - k0):
                    np.minimum(low, lx[i][:, k:k + 1] + lw[j][None, :, k], out=low)
            ok = np.isfinite(low)
            if ok.any():
                worst = max(worst, float((s[ok] / np.exp2(low[ok])).max()))
    return worst


def fwd_budget(a, w, c=None):
    n_rep = 1 if c is None else c.shape[1]
    xh, xl = split(scaled_steps(a, c))
    wh, wl = split(weight_steps(w, n_rep))
    return chain_budget(xh, xl, wh, wl, _groups(xh.shape[1] // LIN_BK, None))


def bwd_data_budget(gy, w, c=None):
    o = w.shape[0]
    n_rep = 1 if c is None else c.shape[1]
    xh, xl = split(scaled_steps(gy, c))
    wr = weight_steps(reblock_weight(w, n_rep), n_rep)
    wh, wl = split(wr)
    fold = LIN_FOLD_STEPS if bwd_data_fold(o, n_rep) else None
    return chain_budget(xh, xl, wh, wl, _groups(xh.shape[1] // LIN_BK, fold))


def bwd_weight_budget(gy, a, c=None):
    n, o = gy.shape
    n_rep = 1 if c is None else c.shape[1]
    ap = np.asarray(a, F32) if c is None else np.concatenate([a * c[:, s:s + 1] for s in range(n_rep)], axis=1)
    yh, yl = split(gy)
    ah, al = split(ap)
    _, _, n_split, rows = bwd_weight_plan(n, ap.shape[1], o)
    worst = 0.0
    pad = lambda m: np.pad(m, ((0, 0), (0, (-m.shape[1]) % LIN_BK)))
    for sp in range(n_split):
        r0, r1 = sp * rows, min(n, (sp + 1) * rows)
        for g0 in range(r0, r1, WG_FOLD_ROWS):
            g1 = min(g0 + WG_FOLD_ROWS, r1)
            sl = slice(g0, g1)
            worst = max(worst, chain_budget(pad(yh[sl].T), pad(yl[sl].T), pad(ah[sl].T), pad(al[sl].T),
                                            [(0, -(-(g1 - g0) // LIN_BK))]))
    return worst


# ---- the GPU cases (shared with the host file, which proves their grid data tells the alternatives apart) -------------
# forward: (n, k, n_scalers (0: pna_linear_fwd), o, bias).  kM = 128 (O <= 128) / 64, kAhead = 2 / 4, kSt = 3 / 2.
FWD_CASES = [
    (1, 32, 0, 64, True),        # N = 1, n_kb = 1, n_it < kSt
    (127, 64, 0, 64, False),     # kM - 1, n_kb = kAhead
    (128, 96, 3, 64, True),      # kM, n_kb = kAhead + 1, n_it = 9 > 2 kSt (the ring wraps with both parities)
    (129, 32, 3, 64, False),     # kM + 1, n_it = kSt
    (300, 64, 2, 128, True),     # n_it = 4
    (513, 32, 5, 128, True),     # S = 5, several tiles
    (128, 96, 0, 128, False),    # n_it = kSt
    (1000, 160, 4, 128, True),   # n_it = 20
    (63, 32, 0, 256, True),      # O = 256: kM - 1, n_it = 1 < kSt
    (64, 96, 0, 256, False),     # kM, n_kb = kAhead - 1, n_it > kSt
    (65, 128, 0, 256, True),     # kM + 1, n_kb = kAhead, n_it = 2 kSt
    (200, 160, 3, 256, True),    # n_kb = kAhead + 1, n_it = 15
    (130, 32, 2, 256, False),    # n_it = kSt
]
# data gradient: (n, n_cols, o, n_scalers).  n_it = O S / 32.
BWD_DATA_CASES = [
    (130, 96, 128, 0),           # n_it = 4: no FOLD; slab 128, one narrow slab (n_cols % 128 = 96)
    (129, 64, 64, 0),            # n_it = 2: no FOLD; slab 64, one slab
    (200, 192, 64, 3),           # n_it = 6: FOLD with a short final chain; three 64-slabs (n_cols % 128 = 64)
    (257, 160, 64, 5),           # n_it = 10: short final chain; 64-slabs, the last 32 wide
    (300, 352, 128, 2),          # n_it = 8: the last fold skipped; 128-slabs, the last 96 wide
    (700, 224, 256, 5),          # n_it = 40; two 128-slabs, the last 96 wide
]
# weight gradient: (n, n_a, o, n_scalers)
BWD_WEIGHT_CASES = [
    (100, 64, 64, 0),            # one split, odd last fold (36 rows); O = 64: warpgroup 1 entirely past n_in = 64
    (40, 32, 128, 0),            # one split of one short fold
    (1500, 96, 64, 3),           # 3 splits of 512 rows, the last 476 (odd last fold); n_in % 128 = 32
    (2000, 32, 128, 3),          # 4 splits; n_in = 96
    (700, 64, 256, 2),           # O = 256: two o_tiles; 2 splits of 352 rows (an odd last fold in each)
]


def fwd_case_data(case, seed=0):
    n, k, s_n, o, bias = case
    return grid_fwd(seed + n * 7 + k + o + s_n, n, k, o, s_n, bias)


def bwd_data_case_data(case, seed=0):
    n, n_cols, o, s_n = case
    return grid_bwd_data(seed + n * 7 + n_cols + o + s_n, n, n_cols, o, s_n)


def bwd_weight_case_data(case, seed=0):
    n, n_a, o, s_n = case
    return grid_bwd_weight(seed + n * 7 + n_a + o + s_n, n, n_a, o, s_n)


def alternatives(kind, case):
    """The restatement's alternatives a case's data must tell apart from it (those its shape can reach)."""
    alts = {"lolo": dict(lolo=True), "rz": dict(mode="rz")}
    if kind == "fwd":
        if case[2]:
            alts["scale_after"] = dict(scale_after=True)
    elif kind == "bwd_data":
        n, n_cols, o, s_n = case
        if s_n:
            alts["scale_after"] = dict(scale_after=True)
        n_it = o * max(s_n, 1) // LIN_BK
        for f in (3, 5, None):
            stated = LIN_FOLD_STEPS if bwd_data_fold(o, max(s_n, 1)) else None
            if _groups(n_it, f) != _groups(n_it, stated):
                alts[f"fold{f}"] = dict(fold=f)
    else:
        n, n_a, o, s_n = case
        if s_n:
            alts["scale_after"] = dict(scale_after=True)
        _, _, n_split, rows = bwd_weight_plan(n, n_a * max(s_n, 1), o)
        sizes = [min(rows, n - r0) for r0 in range(0, n, rows)]
        for steps in (3, 5):
            f = steps * LIN_BK
            if any(-(-m // f) != -(-m // WG_FOLD_ROWS) or m > WG_FOLD_ROWS for m in sizes):
                alts[f"fold{steps}"] = dict(fold_rows=f)
        if n_split > 2:
            alts["desc"] = dict(order="desc")
    return alts
