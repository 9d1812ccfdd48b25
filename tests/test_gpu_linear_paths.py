"""The tensor-core linear (pna_linear.cu) against its exact restatement (tests/linear_paths_ref.py), on the GPU.

Every case names the instance it reaches and calls the C ABI directly, with pitched operands (lda > K, ld_grad_y > O) whose
pitch gaps and spare rows hold NaN the kernels must not read, and outputs whose pitch gaps and spare rows hold a sentinel
bit pattern the kernels must not write.  The outputs start as NaN.
  * Exact tier: on grid data the output equals the restatement bit for bit (NaN where NaN).  The host file proves that on
    the same data the restatement differs from every alternative (fold periods, split order, lo.lo, a truncating split,
    scaling after the split), so the probe of each case is which restatement matched.
  * Bar tier: randn operands and pna_row_scales factors, elementwise within (m + 1) 2^-23 sum|terms| per chain plus the
    final roundings of the exactly summed restatement.
  * Non-finite and extreme operands: NaN rows, infinities, values within 2^-11 of FLT_MAX, 2^+-100, subnormal lo parts.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import linear_paths_ref as R

pytestmark = pytest.mark.gpu
F32 = np.float32
SENTINEL = 0x7F8ACAFE          # a signalling-NaN pattern no float operation produces
# What the tensor cores do with a subnormal lo part (an input near 2^-120), measured on an H100: they keep subnormal operands
# and products (no flush to zero).  DESIGN.md states it beside the split.
SUBNORMAL_MODEL = "kept"


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def L():
    from pna_b200 import _lib
    return _lib.lib()


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(L, rc):
    assert rc == 0, L.pna_last_error()


def pitched_input(x, pad_cols=4, spare_rows=3):
    """x [N, K] on the GPU inside a [N + spare, K + pad] NaN buffer: (view, pitch)."""
    n, k = x.shape
    buf = torch.full((n + spare_rows, k + pad_cols), float("nan"), device=dev())
    buf[:n, :k] = torch.from_numpy(np.ascontiguousarray(x)).to(dev())
    return buf, k + pad_cols


def pitched_output(n, k, pad_cols=8, spare_rows=3):
    """[N + spare, K + pad] with the sentinel everywhere and NaN in the [N, K] output: (buffer, pitch)."""
    buf = torch.full((n + spare_rows, k + pad_cols), SENTINEL, dtype=torch.int32, device=dev()).view(torch.float32)
    buf[:n, :k] = float("nan")
    return buf, k + pad_cols


def check_sentinels(buf, n, k):
    b = buf.view(torch.int32)
    assert bool((b[:n, k:] == SENTINEL).all()), "a store landed in the pitch gap"
    assert bool((b[n:] == SENTINEL).all()), "a store landed in a row past N"


def exact_equal(got, want):
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    nan_g, nan_w = np.isnan(got), np.isnan(want)
    assert np.array_equal(nan_g, nan_w), f"NaN at {np.argwhere(nan_g != nan_w)[:5].tolist()}"
    ok = nan_g | (got == want)
    bad = np.argwhere(~ok)
    assert bad.size == 0, f"{bad.shape[0]} elements differ, first {bad[:3].tolist()}: " + \
        ", ".join(f"{got[tuple(i)]!r} vs {want[tuple(i)]!r}" for i in bad[:3])


def tensor(x):
    return None if x is None else torch.from_numpy(np.ascontiguousarray(x, dtype=F32)).to(dev())


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


# ---- launchers through the ABI ---------------------------------------------------------------------------------------
def run_fwd(L, a, w, b, c, pad_a=4, pad_y=8):
    n, k = a.shape
    o = w.shape[0]
    s_n = 1 if c is None else c.shape[1]
    abuf, lda = pitched_input(a, pad_a)
    ybuf, ldy = pitched_output(n, o, pad_y)
    wd, bd, cd = tensor(w), tensor(b), tensor(c)
    ws = torch.empty(R.fwd_workspace_bytes(k * s_n, o) // 4, device=dev())
    if c is None:
        rc = L.pna_linear_fwd(ptr(abuf), lda, ptr(wd), ptr(bd), ptr(ybuf), ldy, n, k, o, ptr(ws), ws.numel() * 4, _stream())
    else:
        rc = L.pna_linear_scaled_fwd(ptr(abuf), lda, ptr(cd), s_n, ptr(wd), ptr(bd), ptr(ybuf), ldy, n, k * s_n, o, ptr(ws),
                                     ws.numel() * 4, _stream())
    _check(L, rc)
    torch.cuda.synchronize()
    check_sentinels(ybuf, n, o)
    return ybuf[:n, :o].cpu().numpy()


def run_bwd_data(L, gy, w, c, pad_y=4, pad_a=36):
    n, o = gy.shape
    s_n = 1 if c is None else c.shape[1]
    n_in = w.shape[1]
    n_cols = n_in // s_n
    ybuf, ldy = pitched_input(gy, pad_y)
    abuf, lda = pitched_output(n, n_cols, pad_a)
    wd, cd = tensor(w), tensor(c)
    ws = torch.empty(R.bwd_workspace_bytes(n, n_in, o, s_n) // 4 + 4, device=dev())
    _check(L, L.pna_linear_bwd_data(ptr(ybuf), ldy, ptr(cd), s_n, ptr(wd), ptr(abuf), lda, n, n_in, o, ptr(ws), ws.numel() * 4,
                                    _stream()))
    torch.cuda.synchronize()
    check_sentinels(abuf, n, n_cols)
    return abuf[:n, :n_cols].cpu().numpy()


def run_bwd_weight(L, gy, a, c, pad_y=4, pad_a=4):
    n, o = gy.shape
    s_n = 1 if c is None else c.shape[1]
    n_in = a.shape[1] * s_n
    ybuf, ldy = pitched_input(gy, pad_y)
    abuf, lda = pitched_input(a, pad_a)
    cd = tensor(c)
    out = torch.full((o * n_in + 64,), SENTINEL, dtype=torch.int32, device=dev()).view(torch.float32)
    out[:o * n_in] = float("nan")
    ws = torch.empty(max(R.bwd_workspace_bytes(n, n_in, o, s_n) // 4, 4), device=dev())
    _check(L, L.pna_linear_bwd_weight(ptr(ybuf), ldy, ptr(abuf), lda, ptr(cd), s_n, ptr(out), n, n_in, o, ptr(ws),
                                      ws.numel() * 4, _stream()))
    torch.cuda.synchronize()
    assert bool((out.view(torch.int32)[o * n_in:] == SENTINEL).all()), "a store landed past dW"
    return out[:o * n_in].view(o, n_in).cpu().numpy()


# ---- exact tier ------------------------------------------------------------------------------------------------------
def _fwd_id(case):
    n, k, s_n, o, bias = case
    return f"k_linear_3xtf32<{o}>-N{n}-K{k}-S{s_n}-{'bias' if bias else 'nobias'}"


@pytest.mark.parametrize("case", R.FWD_CASES, ids=_fwd_id)
def test_forward_exact(L, case):
    a, w, b, c = R.fwd_case_data(case)
    y = run_fwd(L, a, w, b, c)
    exact_equal(y, R.fwd_restate(a, w, b, c))
    for name, kw in R.alternatives("fwd", case).items():      # probe: the stated restatement, and no alternative, matched
        assert not np.array_equal(y, R.fwd_restate(a, w, b, c, **kw)), name


def _bd_id(case):
    n, n_cols, o, s_n = case
    os_, n_slabs, last = R.bwd_data_slabs(n_cols)
    fold = R.bwd_data_fold(o, max(s_n, 1))
    return f"k_linear_3xtf32<{os_},FOLD={str(fold).lower()}>-N{n}-cols{n_cols}-O{o}-S{s_n}-slabs{n_slabs}x{os_}-last{last}"


@pytest.mark.parametrize("case", R.BWD_DATA_CASES, ids=_bd_id)
def test_bwd_data_exact(L, case):
    gy, w, c = R.bwd_data_case_data(case)
    g = run_bwd_data(L, gy, w, c)
    exact_equal(g, R.bwd_data_restate(gy, w, c))
    for name, kw in R.alternatives("bwd_data", case).items():
        assert not np.array_equal(g, R.bwd_data_restate(gy, w, c, **kw)), name


def _bw_id(case):
    n, n_a, o, s_n = case
    ct, ot, ns, rows = R.bwd_weight_plan(n, n_a * max(s_n, 1), o)
    return f"k_linear_bwd_weight<{o}>-N{n}-nin{n_a * max(s_n, 1)}-splits{ns}x{rows}-otiles{ot}"


@pytest.mark.parametrize("case", R.BWD_WEIGHT_CASES, ids=_bw_id)
def test_bwd_weight_exact(L, case):
    gy, a, c = R.bwd_weight_case_data(case)
    g = run_bwd_weight(L, gy, a, c)
    exact_equal(g, R.bwd_weight_restate(gy, a, c))
    for name, kw in R.alternatives("bwd_weight", case).items():
        assert not np.array_equal(g, R.bwd_weight_restate(gy, a, c, **kw)), name


# ---- bar tier --------------------------------------------------------------------------------------------------------
def row_scales(L, n, s_n, seed):
    """Real factors: pna_row_scales of a seeded in-degree sequence (zeros included), scalers from the five known ones."""
    rng = np.random.default_rng(seed)
    deg = rng.integers(0, 40, n).astype(np.int32)
    deg[: max(1, n // 20)] = 0
    rowptr = torch.from_numpy(np.concatenate([[0], np.cumsum(deg)]).astype(np.int32)).to(dev())
    codes = sum(((s % 5) << (4 * s)) for s in range(s_n))
    avg_log = float(np.mean(np.log(deg.astype(np.float64) + 1)))
    avg_lin = float(np.mean(deg))
    out = torch.empty(n, s_n, device=dev())
    _check(L, L.pna_row_scales(ptr(rowptr), n, s_n, codes, C.c_float(avg_log), C.c_float(avg_lin), ptr(out), _stream()))
    torch.cuda.synchronize()
    return out.cpu().numpy()


def within_bar(got, want, bar, n_adds):
    lim = bar + R.rounding_slack(want, n_adds) + np.abs(want.astype(np.float64)) * 2.0 ** -40
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert np.isfinite(got).all()
    worst = float(np.max(d / np.maximum(lim, 1e-300)))
    assert worst <= 1.0, f"error {worst:.3f} x the bar"
    return worst


@pytest.mark.parametrize("case", R.FWD_CASES, ids=_fwd_id)
def test_forward_bar(L, case):
    n, k, s_n, o, bias = case
    rng = np.random.default_rng(n + k + o)
    a = rng.standard_normal((n, k)).astype(F32)
    w = (rng.standard_normal((o, k * max(s_n, 1))) / np.sqrt(k * max(s_n, 1))).astype(F32)
    b = rng.standard_normal(o).astype(F32) if bias else None
    c = row_scales(L, n, s_n, n + k) if s_n else None
    y = run_fwd(L, a, w, b, c)
    want, bar = R.fwd_restate(a, w, b, c, bars=True)
    within_bar(y, want, bar, 2)


@pytest.mark.parametrize("case", R.BWD_DATA_CASES, ids=_bd_id)
def test_bwd_data_bar(L, case):
    n, n_cols, o, s_n = case
    rng = np.random.default_rng(n + n_cols)
    gy = rng.standard_normal((n, o)).astype(F32)
    w = (rng.standard_normal((o, n_cols * max(s_n, 1))) / np.sqrt(n_cols)).astype(F32)
    c = row_scales(L, n, s_n, n) if s_n else None
    g = run_bwd_data(L, gy, w, c)
    want, bar = R.bwd_data_restate(gy, w, c, bars=True)
    within_bar(g, want, bar, 2 * (o * max(s_n, 1) // 128 + 1))


@pytest.mark.parametrize("case", R.BWD_WEIGHT_CASES, ids=_bw_id)
def test_bwd_weight_bar(L, case):
    n, n_a, o, s_n = case
    rng = np.random.default_rng(n + n_a + o)
    gy = rng.standard_normal((n, o)).astype(F32)
    a = rng.standard_normal((n, n_a)).astype(F32)
    c = row_scales(L, n, s_n, n + 1) if s_n else None
    g = run_bwd_weight(L, gy, a, c)
    want, bar = R.bwd_weight_restate(gy, a, c, bars=True)
    within_bar(g, want, bar, 2 * (n // 64 + 2))


@pytest.mark.parametrize("shift", [-100, 100])
def test_forward_far_from_one_stays_within_the_bar(L, shift):
    rng = np.random.default_rng(11)
    a = (rng.standard_normal((200, 96)) * 2.0 ** shift).astype(F32)
    w = (rng.standard_normal((128, 192)) / 14).astype(F32)
    c = row_scales(L, 200, 2, 12)
    y = run_fwd(L, a, w, None, c)
    want, bar = R.fwd_restate(a, w, None, c, bars=True)
    within_bar(y, want, bar, 2)


# ---- non-finite and extreme operands ---------------------------------------------------------------------------------
def test_nan_row_poisons_its_row_only(L):
    a, w, b, c = R.fwd_case_data((300, 64, 2, 128, True))
    a[7, 3] = np.nan
    y = run_fwd(L, a, w, b, c)
    assert np.isnan(y[7]).all() and not np.isnan(np.delete(y, 7, axis=0)).any()
    exact_equal(y, R.fwd_restate(a, w, b, c))


def test_infinities_give_what_fp32_gives(L):
    """inf * w = +-inf, inf * 0 and inf - inf = NaN.  Before hi was rounded with satfinite, an inf split into hi = inf and
    lo = NaN and every output of its row was NaN."""
    a, w, b, c = R.fwd_case_data((130, 64, 0, 128, True))
    w[:5, 4] = 0                                             # inf * 0 in outputs 0..4
    w[5:, 4][w[5:, 4] == 0] = F32(0.0625)
    a[9, 4] = np.inf
    a[10, 4] = -np.inf
    a[11, 4], a[11, 6] = np.inf, np.inf                      # inf - inf where w[:, 4] and w[:, 6] differ in sign
    y = run_fwd(L, a, w, b, c)
    with np.errstate(invalid="ignore", over="ignore"):
        fp32 = a.astype(np.float64) @ w.T.astype(np.float64) + b
    for r in (9, 10, 11):
        assert np.array_equal(np.isnan(y[r]), np.isnan(fp32[r])), r
        fin = ~np.isnan(fp32[r])
        assert np.array_equal(y[r][fin], fp32[r][fin].astype(F32)), r
    assert np.isnan(y[11]).any() and np.isinf(y[11]).any() and np.isnan(y[9, :5]).all() and np.isinf(y[9, 5:]).all() and np.isinf(y[10, 5:]).all()
    exact_equal(y, R.fwd_restate(a, w, b, c))


@pytest.mark.parametrize("o", [64, 256])
def test_near_flt_max_stays_finite(L, o):
    """Finite |x| >= 0x7F7FF000 rounds to inf under cvt.rna; the split keeps hi finite (satfinite) and the result stays
    within the bar."""
    rng = np.random.default_rng(o)
    a = rng.standard_normal((70, 64)).astype(F32)
    big = np.array([0x7F7FF000, 0x7F7FFFFF, 0xFF7FF800, 0x7F7FEFFF], dtype=np.uint32).view(F32)
    a[3, :4] = big
    a[40, 10:14] = -big
    w = (rng.standard_normal((o, 64)) * 2.0 ** -12).astype(F32)
    y = run_fwd(L, a, w, None, None)
    assert np.isfinite(y).all()
    assert not np.isfinite(R.fwd_restate(a, w, mode="rna_unsat")).all()   # what the unsaturated split gave
    want, bar = R.fwd_restate(a, w, None, None, bars=True)
    within_bar(y, want, bar, 2)


def subnormal_models():
    """A row whose only nonzero is x = 2^-120 + 2^-132 (hi normal, lo subnormal) against w = 1 + 2^-14: the terms are
    hi.hi = 2^-120, hi.lo = 2^-134 (a subnormal product of normal operands) and lo.hi = 2^-132 (a subnormal operand).
    The models keep everything, flush subnormal operands, or flush subnormal products (or the subnormal chain sum)."""
    x = F32(2.0 ** -120 + 2.0 ** -132)
    w = F32(1.0 + 2.0 ** -14)
    hh, hl, lh = 2.0 ** -120, 2.0 ** -134, 2.0 ** -132
    return x, w, {"kept": F32(F32(hh) + F32(hl + lh)), "operands_flushed": F32(F32(hh) + F32(hl)),
                  "products_flushed": F32(hh)}


def test_subnormal_lo_parts(L, record_property):
    x, w1, models = subnormal_models()
    assert len(set(float(v) for v in models.values())) == 3
    a = np.zeros((64, 32), F32)
    a[5, 2] = x
    w = np.zeros((64, 32), F32)
    w[:, 2] = w1
    y = run_fwd(L, a, w, None, None)
    got = y[5, 0]
    assert np.all(y[5] == got) and not np.any(np.delete(y, 5, axis=0))
    seen = [k for k, v in models.items() if v == got]
    record_property("subnormal_model", seen)
    print(f"subnormal lo parts: y = {float(got)!r} -> {seen}")
    assert seen, f"{float(got)!r} matches no model: {models}"
    if SUBNORMAL_MODEL is not None:
        assert seen == [SUBNORMAL_MODEL]


def test_rows_past_4_gib(L):
    """A's last rows more than 4 GiB from its base, reached through a large pitch."""
    free, _ = torch.cuda.mem_get_info(dev())
    if free < 16 * 2 ** 30:
        pytest.skip(f"needs 16 GiB of free device memory for a 4.6 GB operand, {free / 2 ** 30:.1f} free")
    a, w, b, c = R.fwd_case_data((130, 64, 0, 64, True))
    n, k = a.shape
    lda = ((int(4.3 * 2 ** 30) // 4) // (n - 1) + 3) // 4 * 4
    big = torch.empty((n - 1) * lda + k, device=dev())
    view = big.as_strided((n, k), (lda, 1))
    view.copy_(torch.from_numpy(a).to(dev()))
    assert (n - 1) * lda * 4 > 4 * 2 ** 30
    ybuf, ldy = pitched_output(n, 64)
    ws = torch.empty(R.fwd_workspace_bytes(k, 64) // 4, device=dev())
    wd, bd = tensor(w), tensor(b)
    _check(L, L.pna_linear_fwd(ptr(big), lda, ptr(wd), ptr(bd), ptr(ybuf), ldy, n, k, 64, ptr(ws), ws.numel() * 4, _stream()))
    torch.cuda.synchronize()
    check_sentinels(ybuf, n, 64)
    exact_equal(ybuf[:n, :64], R.fwd_restate(a, w, b, c))
    del big, view
    torch.cuda.empty_cache()
