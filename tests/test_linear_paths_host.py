"""Host checks of tests/linear_paths_ref.py, the restatement of the tensor-core linear (CPU only).

* tf32_rna against an independent Fraction rounding (ties away from zero), on ties, subnormals, the FLT_MAX boundary,
  infinities and NaNs; the split with and without satfinite.
* The restated launch plan against the library's own workspace query (which answers without a GPU).
* The grid data of every GPU case: split gives back the designed parts, every chain meets the 2^12 budget, and the stated
  restatement differs in bits from every alternative the case can reach, so the GPU tests can tell them apart.
* On integer data every grouping of the chains agrees with the others and with float64.
"""
import ctypes as C
from fractions import Fraction

import numpy as np
import pytest

import linear_paths_ref as R

F32 = np.float32


def bits(x):
    return np.asarray(x, dtype=F32).view(np.uint32)


def from_bits(b):
    return np.asarray(b, dtype=np.uint32).view(F32)


def tf32_fraction(b: int, satfinite: bool):
    """Round the fp32 value with bits b to 10 explicit mantissa bits, ties away from zero, by exact rational arithmetic."""
    x = Fraction(float(from_bits(np.uint32(b))))
    if x == 0:
        return b & 0x80000000
    sign = -1 if x < 0 else 1
    m = abs(x)
    e = max(m.numerator.bit_length() - m.denominator.bit_length() - (1 if m < 2 ** (m.numerator.bit_length() - m.denominator.bit_length()) else 0), -126)
    q = Fraction(2) ** (e - 10)                        # the TF32 grid of the binade (subnormals: 2^-136)
    k = m / q
    r = int(k) + (1 if k - int(k) >= Fraction(1, 2) else 0)
    v = r * q
    if v >= Fraction(2) ** 128:
        out = F32(np.inf) if not satfinite else from_bits(np.uint32(R.TF32_MAX_BITS))
    else:
        out = F32(float(v))
    return int(bits(F32(sign) * out))


def _samples():
    rng = np.random.default_rng(1)
    b = [rng.integers(0, 2 ** 32, 3000, dtype=np.uint64)]
    mant = rng.integers(0, 2 ** 10, 400, dtype=np.uint64) << 13
    exps = rng.integers(0, 255, 400, dtype=np.uint64) << 23
    b.append(exps | mant | 0x1000)                     # exact ties
    b.append(exps | mant | 0x0FFF)                     # just below a tie
    b.append(rng.integers(1, 0x800000, 400, dtype=np.uint64))    # subnormals
    b.append(np.array([0x7FFFFF, 0x7FF000, 0x7FEFFF, 0x7F7FEFFF, 0x7F7FF000, 0x7F7FF001, 0x7F7FFFFF, 0x7F7FE000, 0,
                       0x00001000, 0x00000FFF], dtype=np.uint64))
    out = np.concatenate(b).astype(np.uint32)
    out = np.concatenate([out, out | np.uint32(0x80000000)])
    return out[(out & 0x7F800000) != 0x7F800000]


@pytest.mark.parametrize("sat", [False, True])
def test_tf32_rna_matches_fraction_rounding(sat):
    s = _samples()
    got = bits(R.tf32_rna(from_bits(s), satfinite=sat))
    want = np.array([tf32_fraction(int(b), sat) for b in s], dtype=np.uint32)
    bad = np.nonzero(got != want)[0]
    assert bad.size == 0, [(hex(s[i]), hex(got[i]), hex(want[i])) for i in bad[:5]]


def test_tf32_non_finite_and_flt_max():
    inf, nan_hi = from_bits(np.uint32(0x7F800000)), from_bits(np.uint32(0x7FC12345))
    assert bits(R.tf32_rna(inf)) == 0x7F800000 and bits(R.tf32_rna(-inf)) == 0xFF800000
    assert bits(R.tf32_rna(nan_hi)) == 0x7FC12345 & 0xFFFFE000                 # mask only: the payload's top bits stay
    assert bits(R.tf32_rna(inf, satfinite=True)) == R.TF32_MAX_BITS
    big = from_bits(np.array([0x7F7FF000, 0xFF7FFFFF, 0x7F7FEFFF], dtype=np.uint32))
    hi, lo = R.split(big, "rna_unsat")                # the split before satfinite: hi = +-inf, lo = -+inf, products NaN
    assert np.isinf(hi[:2]).all() and np.isinf(lo[:2]).all() and np.isfinite(hi[2])
    hi, lo = R.split(big)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    assert np.all(hi.astype(np.float64) + lo.astype(np.float64) - big.astype(np.float64)
                  <= np.abs(big.astype(np.float64)) * 2.0 ** -22)
    hi, lo = R.split(np.array([np.inf, -np.inf], dtype=F32))
    assert (bits(hi) & 0x7FFFFFFF == R.TF32_MAX_BITS).all() and np.array_equal(lo, [np.inf, -np.inf])


def _lib():
    from pna_b200 import _lib
    try:
        return _lib.lib()
    except ImportError as e:
        pytest.skip(str(e))


def test_plan_and_slabs_match_the_library_workspace():
    L = _lib()
    nb = C.c_size_t()
    seen_split = set()
    for o in (64, 128, 256):
        for s_n in (1, 2, 3, 5):
            for n_cols in (32, 64, 96, 128, 160, 192, 224, 352, 1024):
                n_in = n_cols * s_n
                for n in (0, 1, 100, 511, 512, 513, 1500, 4099, 70_000, 1_000_003):
                    assert L.pna_linear_bwd_workspace_bytes(n, n_in, o, s_n, C.byref(nb)) == 0
                    assert nb.value == R.bwd_workspace_bytes(n, n_in, o, s_n), (n, n_in, o, s_n)
                    if n and nb.value > R.bwd_workspace_bytes(0, n_in, o, s_n):    # the partials dominate: n_split shows
                        seen_split.add(R.bwd_weight_plan(n, n_in, o)[2])
                assert L.pna_linear_workspace_bytes(n_in, o, C.byref(nb)) == 0 and nb.value == R.fwd_workspace_bytes(n_in, o)
    assert len(seen_split) >= 5
    assert R.bwd_data_slabs(160) == (64, 3, 32) and R.bwd_data_slabs(352) == (128, 3, 96) and R.bwd_data_slabs(192) == (64, 3, 64)
    assert R.bwd_weight_plan(1500, 288, 64) == (3, 1, 3, 512) and R.bwd_weight_plan(100, 64, 64) == (1, 1, 1, 128)
    assert [R.k_ahead(o) for o in (64, 128, 256)] == [2, 2, 4] and [R.lin_stages(o) for o in (64, 128, 256)] == [3, 3, 2]


def test_grid_parts_split_back():
    rng = np.random.default_rng(3)
    for e, sh in ((-3, 18), (-4, 19), (5, 14), (-100, 13)):
        hi, lo = R.grid_matrix(rng, (64, 96), e, 0.7, lo_shift=sh)
        h, l = R.split(hi + lo)
        assert np.array_equal(h, hi) and np.array_equal(l, lo)
    for v, w in ((R.probe_x(-3), R.probe_w(-4)), (R.probe_scaled_x(-3), R.probe_w(-4))):
        for x in (v, w):
            h, l = R.split(np.array([x]))
            assert l[0] != 0 and abs(float(l[0])) <= abs(float(h[0])) * 2.0 ** -11
    h, l = R.split(np.array([R.probe_scaled_x(-3)]))
    h2, l2 = R.split(np.array([R.probe_scaled_x(-3) * F32(R.PROBE_SCALE)]))
    assert h2[0] != h[0] * F32(R.PROBE_SCALE)                     # the scaled probe splits differently


def _differs(y, z):
    return int(np.count_nonzero(bits(y) != bits(z)))


@pytest.mark.parametrize("case", R.FWD_CASES)
def test_forward_grid_data_tells_the_alternatives_apart(case):
    a, w, b, c = R.fwd_case_data(case)
    assert R.fwd_budget(a, w, c) <= 2 ** 12
    y = R.fwd_restate(a, w, b, c)
    for name, kw in R.alternatives("fwd", case).items():
        assert _differs(y, R.fwd_restate(a, w, b, c, **kw)) > 0, name


@pytest.mark.parametrize("case", R.BWD_DATA_CASES)
def test_bwd_data_grid_data_tells_the_alternatives_apart(case):
    gy, w, c = R.bwd_data_case_data(case)
    assert R.bwd_data_budget(gy, w, c) <= 2 ** 12
    y = R.bwd_data_restate(gy, w, c)
    alts = R.alternatives("bwd_data", case)
    if R.bwd_data_fold(case[2], max(case[3], 1)):
        assert {"fold3", "fold5", "foldNone"} <= set(alts)
    for name, kw in alts.items():
        assert _differs(y, R.bwd_data_restate(gy, w, c, **kw)) > 0, name


@pytest.mark.parametrize("case", R.BWD_WEIGHT_CASES)
def test_bwd_weight_grid_data_tells_the_alternatives_apart(case):
    gy, a, c = R.bwd_weight_case_data(case)
    assert R.bwd_weight_budget(gy, a, c) <= 2 ** 12
    y = R.bwd_weight_restate(gy, a, c)
    for name, kw in R.alternatives("bwd_weight", case).items():
        assert _differs(y, R.bwd_weight_restate(gy, a, c, **kw)) > 0, name


def test_integer_data_all_groupings_agree_with_float64():
    rng = np.random.default_rng(5)
    gy = rng.integers(-3, 4, (700, 64)).astype(F32)
    a = rng.integers(-3, 4, (700, 64)).astype(F32)
    c = rng.integers(0, 3, (700, 3)).astype(F32)
    w = rng.integers(-3, 4, (64, 192)).astype(F32)
    want = gy.astype(np.float64).T @ np.concatenate([a * c[:, s:s + 1] for s in range(3)], 1).astype(np.float64)
    for kw in (dict(), dict(fold_rows=96), dict(fold_rows=160), dict(order="desc")):
        assert np.array_equal(R.bwd_weight_restate(gy, a, c, **kw), want)
    want = sum(c[:, s:s + 1].astype(np.float64) * (gy.astype(np.float64) @ w[:, s * 64:(s + 1) * 64].astype(np.float64))
               for s in range(3))
    for kw in (dict(), dict(fold=3), dict(fold=5), dict(fold=None)):
        assert np.array_equal(R.bwd_data_restate(gy, w, c, **kw), want)
    want = np.concatenate([a * c[:, s:s + 1] for s in range(3)], 1).astype(np.float64) @ w.T.astype(np.float64)
    assert np.array_equal(R.fwd_restate(a, w, None, c), want)


def test_random_bar_covers_float64():
    """On random data the float64 product lies within the restatement's bar (the restatement drops lo.lo, 2^-22 of a
    product at most, which the bar's own rounding terms cover)."""
    rng = np.random.default_rng(9)
    a = rng.standard_normal((300, 128)).astype(F32)
    w = (rng.standard_normal((128, 256)) / 16).astype(F32)
    c = rng.uniform(0, 3, (300, 2)).astype(F32)
    y, bar = R.fwd_restate(a, w, None, c, bars=True)
    exact = np.concatenate([a * c[:, s:s + 1] for s in range(2)], 1).astype(np.float64) @ w.T.astype(np.float64)
    assert np.all(np.abs(y - exact) <= bar + R.rounding_slack(y, 2) + np.abs(exact) * 2.0 ** -21)
