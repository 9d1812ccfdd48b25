"""The add-on aggregators' fp32 restatement (addon_paths_ref.py) against the kernels run on the HOST, bit for bit.

The host build of pna_aggregate_fwd / pna_aggregate_bwd / pna_aggregate_bwd_slots (tests/emu, the same builds as
test_moments_emulated.py / test_weighted_emulated.py) calls libm's powf / expf / logf; the restatement gets the same powf
and expf injected, and the scaler factors of the same logf, so every element must match bit for bit: the forward's add-on
columns (light and split rows, a row of more than 512 chunks, SKIP_LIGHT / SKIP_HUBS / a masked view) and the whole backward
(the core kernels' term, then the add-ons'), per-slot and atomic-with-col == NULL instances, feature slabs, grad_row_bias,
fp32 and bf16.  The restatement must also lie within the float64 bars of moment_bars.py / weighted_bars.py, merge chunks
exactly as a written table says, and use the kernels' fp32 constants.
"""
import ctypes as C
import ctypes.util
import re
import shutil
from fractions import Fraction

import numpy as np
import pytest
import torch

import addon_paths_ref as R
import backward_paths_ref as B
import moment_bars as MB
import weighted_bars as WB
from pna_b200 import _lib
from test_moments_emulated import CHUNK, SCALERS, SPLIT, Case
from test_weighted_emulated import emu  # noqa: F401  (the host build of the add-on kernels, a fixture)

F32 = np.float32
HM = R.host_math()
_LIBM = C.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_LIBM.logf.restype, _LIBM.logf.argtypes = C.c_float, [C.c_float]


def host_scales(c: Case):
    """[N, S] factors of deg_scales with the host's logf (what the host build multiplies by), at the scalers' degree"""
    d = (c.sdeg if c.sdeg is not None else c.deg).numpy().astype(F32)
    lg = np.array([_LIBM.logf(float(v)) for v in d + F32(1)], F32)
    al, an = F32(c.avg["log"]), F32(c.avg["lin"])
    iso = d == 0
    one = np.ones_like(d)
    with np.errstate(divide="ignore"):
        f = {"identity": one, "amplification": lg / al, "attenuation": np.where(iso, one, al / lg), "linear": d / an,
             "inverse_linear": np.where(iso, one, an / d)}
    return np.stack([f[s] for s in c.scalers], 1).astype(F32)


def np32(t):
    return None if t is None else t.float().numpy()


def graph_of(c: Case, col=True, dcol=None):
    return R.Graph(c.rowptr.numpy(), c.col.numpy() if col else None, c.hub_info.numpy(), CHUNK, SPLIT, dcol=dcol)


def as_dtype(a, dtype):
    """one round-to-nearest-even to the output type"""
    return a if dtype == torch.float32 else torch.from_numpy(np.ascontiguousarray(a, F32)).to(torch.bfloat16).float().numpy()


def assert_same(got, want, what=""):
    """bit for bit where the reference is a number, NaN exactly where it is NaN"""
    g, w = np.ascontiguousarray(got, F32), np.ascontiguousarray(want, F32)
    gn, wn = np.isnan(g), np.isnan(w)
    assert (gn == wn).all(), f"{what}: NaN positions differ at {np.argwhere(gn != wn)[:4].tolist()}"
    bad = g.view(np.uint32)[~gn] != w.view(np.uint32)[~wn]
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ"


MIX6 = ("moment4", "softmin", "mean", "normalised_mean", "moment3", "softmax")


def reference_forward(c: Case, flags=0, ldeg=None):
    has_self = c.self_feat is not None
    want = R.forward(graph_of(c), np32(c.x), np32(c.bias), list(c.aggrs), host_scales(c), HM, towers=c.towers,
                     has_self=has_self, flags=flags, ldeg=ldeg)
    return as_dtype(want, c.dtype)


@pytest.mark.parametrize("F,towers,dtype,bias,self_feat,sdeg,aggrs", [
    (12, 1, torch.float32, True, False, False, MIX6),
    (16, 2, torch.float32, False, True, True, MIX6),
    (24, 3, torch.bfloat16, True, True, False, MIX6),
    (10, 1, torch.float32, True, False, True, ("moment5", "moment3", "moment4")),
    (8, 2, torch.bfloat16, False, False, True, ("normalised_mean", "softmax", "softmin")),
])
def test_forward_columns_bit_for_bit(emu, F, towers, dtype, bias, self_feat, sdeg, aggrs):   # noqa: F811
    c = Case(emu, 60, 400, F, seed=F + towers, dtype=dtype, towers=towers, bias=bias, self_feat=self_feat, sdeg=sdeg,
             scalers=SCALERS, aggrs=aggrs)
    assert c.hub_info.size(0) >= 1 and (c.deg == 0).sum() >= 5
    assert_same(c.forward().float().numpy(), reference_forward(c), "forward")
    # PNA_FLAG_ZERO_ISOLATED: rows without in-edges are 0 for every scaler (also where a factor is not 1)
    assert_same(c.forward(flags=_lib.FLAG_ZERO_ISOLATED).float().numpy(), reference_forward(c, flags=R.FLAG_ZERO_ISOLATED))


def test_forward_split_row_with_more_than_512_chunks(emu):   # noqa: F811
    c = Case(emu, 40, 150, 4, seed=3, big=40, huge=CHUNK * 520 + 3, aggrs=("moment3", "softmax", "normalised_mean", "moment5"),
             scalers=("identity", "linear"))
    assert int(c.hub_info[:, 2].max()) > 512
    assert_same(c.forward().float().numpy(), reference_forward(c), "forward, > 512 chunks")


def test_forward_row_selection(emu):   # noqa: F811
    c = Case(emu, 60, 400, 12, seed=8, aggrs=MIX6)
    for fl in (_lib.FLAG_SKIP_LIGHT, _lib.FLAG_SKIP_HUBS):
        assert_same(c.forward(fl).float().numpy(), reference_forward(c, flags=fl), f"flags {fl}")
    mask = torch.arange(c.n) % 2 == 0
    ldeg = torch.where(mask & (c.deg < SPLIT), c.deg, torch.full_like(c.deg, -1)).numpy()
    assert_same(c.forward(view_mask=mask).float().numpy(), reference_forward(c, ldeg=ldeg), "masked view")


# ---- backward -----------------------------------------------------------------------------------------------------------
def run_bwd(c: Case, go, mode, f0=0, fc=None):
    """mode "slots": pna_aggregate_bwd_slots into [E, fc]; "per_slot": pna_aggregate_bwd with col == NULL over the
    messages in CSR order (normalised_mean reads degree_col); outputs start as NaN"""
    fc = c.F - f0 if fc is None else fc
    E = c.col.numel()
    d = c.desc(scratch_rows=6)
    gb = torch.full((c.n, c.F), float("nan")) if c.bias is not None else None
    go = go.to(c.dtype).contiguous()
    gbp = None if gb is None else gb.data_ptr()
    if mode == "slots":
        gs = torch.full((E, fc), float("nan"))
        assert c.emu.pna_aggregate_bwd_slots(C.byref(d), go.data_ptr(), c.W, f0, fc, gs.data_ptr(), fc, gbp, c.F, None) == 0, \
            c.emu.emu_last_error()
        return gs.numpy(), None if gb is None else gb.numpy()
    xm = c.x[c.col.long()].contiguous()
    dcol = c.col.clone()
    gg = torch.full((E, c.F), float("nan"))
    d.gathered, d.col, d.degree_col = xm.data_ptr(), None, dcol.data_ptr()
    assert c.emu.pna_aggregate_bwd(C.byref(d), go.data_ptr(), c.W, gg.data_ptr(), c.F, gbp, c.F, None) == 0, c.emu.emu_last_error()
    return gg.numpy(), None if gb is None else gb.numpy()


def reference_backward(c: Case, go, col=True):
    g = graph_of(c) if col else graph_of(c, col=False, dcol=c.col.numpy())
    x = np32(c.x) if col else np32(c.x)[c.col.long().numpy()]
    return R.backward(g, x, np32(c.bias), go.to(c.dtype).float().numpy(), list(c.aggrs), host_scales(c), HM, towers=c.towers,
                      has_self=c.self_feat is not None)


@pytest.mark.parametrize("F,towers,dtype,bias,self_feat,aggrs", [
    (12, 1, torch.float32, True, False, MIX6),
    (16, 2, torch.float32, True, True, ("softmax", "moment5", "max", "softmax", "std", "moment5")),    # repeated add-ons
    (8, 1, torch.float32, True, False, ("normalised_mean", "softmin", "moment3")),                    # add-ons only
    (24, 3, torch.bfloat16, True, True, MIX6),
    (16, 1, torch.bfloat16, False, False, ("moment4", "normalised_mean", "var")),
    (12, 1, torch.float32, True, False, ("moment5", "sum", "moment3", "softmax", "moment4")),   # c0 over three orders
])
def test_backward_bit_for_bit(emu, F, towers, dtype, bias, self_feat, aggrs):   # noqa: F811
    c = Case(emu, 60, 400, F, seed=30 + F, dtype=dtype, towers=towers, bias=bias, self_feat=self_feat, aggrs=aggrs,
             scalers=("identity", "attenuation", "linear"))
    go = torch.randn(c.n, c.W, generator=torch.Generator().manual_seed(F))
    gs_w, gb_w, _ = reference_backward(c, go)
    gs, gb = run_bwd(c, go, "slots")
    assert_same(gs, gs_w, "grad_slots")
    if bias:
        assert_same(gb, gb_w, "grad_row_bias (per-slot instance)")
    al = 4 if dtype == torch.float32 else 8            # a slab with f0 > 0, and the ragged last one
    gs2, gb2 = run_bwd(c, go, "slots", f0=al, fc=al)
    assert_same(gs2, gs_w[:, al:2 * al], "grad_slots slab")
    if bias:
        assert_same(gb2[:, al:2 * al], gb_w[:, al:2 * al], "grad_row_bias slab")
        assert np.isnan(np.delete(gb2, np.s_[al:2 * al], axis=1)).all()
    last = (F - 1) // al * al
    assert_same(run_bwd(c, go, "slots", f0=last)[0], gs_w[:, last:], "last slab")
    # the atomic instance with col == NULL (messages in CSR order, normalised_mean through degree_col): plain adds, exact
    gg_w, gbp_w, _ = reference_backward(c, go, col=False)
    assert_same(gs_w, gg_w, "the per-slot layout restates the same values")
    gg, gbp = run_bwd(c, go, "per_slot")
    assert_same(gg, gg_w, "grad_gathered (col == NULL)")
    if bias:
        light = ~graph_of(c).hub
        assert_same(gbp[light], gbp_w[light], "grad_row_bias, light rows (atomic instance)")
        if all(R.code_of(a) is not None for a in aggrs):   # no core term: the core's atomic chunk shares are all 0
            assert_same(gbp, gbp_w, "grad_row_bias (atomic instance, add-ons only)")


def test_restatement_within_the_float64_bars(emu):   # noqa: F811
    """Forward values and per-slot gradients of the restatement against moment_bars / weighted_bars on the same messages"""
    c = Case(emu, 60, 400, 12, seed=5, aggrs=("moment3", "moment4", "moment5", "softmax", "softmin", "normalised_mean"),
             scalers=("identity",))
    g = graph_of(c)
    x, b = np32(c.x), np32(c.bias)
    sc = host_scales(c)
    out = R.forward(g, x, b, list(c.aggrs), sc, HM)
    msg = c.messages()
    order = torch.sort(c.dst, stable=True).indices
    for a, name in enumerate(c.aggrs):
        y = torch.from_numpy(out[:, a * c.F:(a + 1) * c.F]).double()
        want, tol = MB.moment_bar(msg, c.dst, c.n, int(name[-1])) if name.startswith("moment") else \
            WB.bar(name, msg, c.dst, c.n, wsrc=c.src)
        assert ((y - want).abs() <= tol).all(), name
    go = torch.randn(c.n, c.W, generator=torch.Generator().manual_seed(1))
    gon = go.numpy()
    m = g.messages(x, b)
    Ft, _, base = R.layout(c.F, 1, False, len(c.aggrs), 1)
    G = {k: torch.from_numpy(gon[:, (k - 3) * c.F:(k - 2) * c.F]) for k in (3, 4, 5)}
    g64, tol = MB.moment_grad_bar(msg, c.dst, c.n, [3, 4, 5], G)
    t, _ = R.moment_terms(g, m, gon, list(c.aggrs), sc, base, Ft, HM)
    assert ((torch.from_numpy(t).double() - g64[order]).abs() <= tol[order]).all(), "moments"
    for a, name in enumerate(c.aggrs[3:], 3):
        Gn = torch.from_numpy(gon[:, a * c.F:(a + 1) * c.F])
        g64, tol = WB.grad_bar(name, msg, c.dst, c.n, Gn, wsrc=c.src)
        t = R.weighted_terms(g, m, gon, list(c.aggrs), sc, base, Ft, name, HM)
        assert ((torch.from_numpy(t).double() - g64[order]).abs() <= tol[order]).all(), name


# ---- hand-built chunk tables ------------------------------------------------------------------------------------------------
def test_chunk_merges_follow_the_written_table():
    """Row 0: 5 slots in chunks of 2 (a split row), messages [2^24, 1, 1, -2^24, 1].  The kernels' sums:
         chunk 0: (0 + 2^24) + 1 = 2^24 (the 1 is lost),  chunk 1: (0 + 1) + -2^24 = 1 - 2^24,  chunk 2: 0 + 1 = 1
         row:     ((0 + 2^24) + (1 - 2^24)) + 1 = 2       (a slot-order sum gives 1, the exact sum is 3)
       Row 1: 4 slots in chunks of 2, maxima tied across chunks: [3, 7, 7, -1] -> M = 7 in chunks 0 and 1, e = expf(0) = 1
       at both, Z = ((0 + e0) + e1) + ((0 + 1) + e3) chunk by chunk."""
    t24 = F32(2.0 ** 24)
    rowptr = np.array([0, 5, 9])
    hub_info = np.array([[0, 0, 3, 5], [1, 3, 2, 4]])
    g = R.Graph(rowptr, np.arange(9), hub_info, 2, 2)
    m = np.array([t24, 1, 1, -t24, 1, 3, 7, 7, -1], F32)[:, None]
    s, shares = g.row_sums(m)
    assert shares[:3, 0].tolist() == [t24, F32(1) - t24, 1]
    assert s[0, 0] == 2 and B.ordered_sums(m, [0], [5])[0, 0] == 1
    assert g.row_max(m)[1, 0] == 7
    y, p = R.weighted_rows(g, m, "softmax", HM)
    e = p["e"][5:, 0]
    assert e[1] == 1 and e[2] == 1
    assert p["Z"][1, 0] == F32(F32(e[0] + e[1]) + F32(F32(1) + e[3]))
    # the order matters: summing the chunk shares in reverse gives another value for a suitable row
    m2 = np.array([1, 0, t24, 0, -t24, 0, 0, 0, 0], F32)[:, None]     # shares 1, 2^24, -2^24: 0 in order, 1 reversed
    s2, sh2 = g.row_sums(m2)
    assert s2[0, 0] == F32(F32(sh2[0, 0] + sh2[1, 0]) + sh2[2, 0]) != F32(F32(sh2[2, 0] + sh2[1, 0]) + sh2[0, 0])


# ---- constants ------------------------------------------------------------------------------------------------------------
def rn32(q: Fraction) -> F32:
    """round-to-nearest-even of a rational to fp32 (normal range)"""
    s = -1 if q < 0 else 1
    q = abs(q)
    e = 0
    while q >= 2 ** (e + 1):
        e += 1
    while q < 2 ** e:
        e -= 1
    scaled = q / Fraction(2) ** (e - 23)
    n, r = divmod(scaled.numerator, scaled.denominator)
    if 2 * r > scaled.denominator or (2 * r == scaled.denominator and n % 2):
        n += 1
    return F32(s * n * 2.0 ** (e - 23))


def test_exponent_constants_match_exact_rounding():
    third = rn32(Fraction(1, 3))
    assert R.INV_K == {3: third, 4: rn32(Fraction(1, 4)), 5: rn32(Fraction(1, 5))}
    # moment_slope's exponent of k = 3 is fl(fl(1/3) - 1): fl(1/3) - 1 needs 25 bits and rounds (a tie, to even), which is
    # not the correctly rounded -2/3
    e3 = rn32(Fraction(float(third)) - 1)
    assert R.SLOPE_E[3] == e3 and e3 != rn32(Fraction(-2, 3)) and Fraction(float(e3)) != Fraction(float(third)) - 1
    assert R.SLOPE_E[4] == rn32(Fraction(-3, 4)) and R.SLOPE_E[5] == rn32(Fraction(-4, 5))


def test_launch_helper():
    A = ["normalised_mean", "mean", "moment4", "softmax"]
    fwd = R.addon_launches(A, 72, 100, 3, 20)
    assert [k for k, _ in fwd] == ["k_mom_rows", "k_mom_chunk_sum<4>", "k_mom_hub_mean<4>", "k_mom_chunk_central<4>",
                                   "k_mom_hub_final", "k_wsum_rows[softmax]", "k_wsum_chunk_max<4>[softmax]", "k_wsum_hub_max<4>",
                                   "k_wsum_chunk_zs<4>[softmax]", "k_wsum_hub_final[softmax]", "k_wsum_rows[normalised_mean]",
                                   "k_wsum_chunk_zs<4>[normalised_mean]", "k_wsum_hub_final[normalised_mean]"]
    assert dict(fwd)["k_mom_rows"] == (13, 3) and dict(fwd)["k_mom_chunk_sum<4>"] == (3, 3) and dict(fwd)["k_mom_hub_mean<4>"] == (1, 3)
    assert [k for k, _ in R.addon_launches(A, 72, 100, 3, 20, flags=R.FLAG_SKIP_LIGHT)] == [k for k, _ in fwd if "rows" not in k]
    bwd = [k for k, _ in R.addon_launches(A, 33, 100, 3, 20, backward=True)]
    assert bwd.count("k_mom_bwd_hub_bias<6>") == 3 and "k_wsum_chunk_zs<6>[normalised_mean]" not in bwd
    assert R.addon_launches(["softmin"], 33, 100, 0, 0, backward=True) == [("k_wsum_bwd_rows[softmin]", (13, 2))]


# ---- the device-math probe ------------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("nvcc") is None, reason="needs nvcc")
def test_devmath_probe_cross_compiles(tmp_path):
    """oracle/devmath builds with the library's nvcc flags, exports its two entry points and includes none of the library's
    headers (a change in the library cannot leak into the oracle)"""
    from oracle import devmath_build
    src = open(devmath_build.SRC).read()
    assert re.findall(r'#include\s*[<"]([^>"]+)', src) == ["cuda_runtime.h"]
    lib = C.CDLL(devmath_build.build(str(tmp_path / "libdevmath_sm90.so"), force=True))
    assert hasattr(lib, "devmath_powf") and hasattr(lib, "devmath_expf")
