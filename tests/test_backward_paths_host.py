"""Checks of the fp32 restatement of the aggregation backward (backward_paths_ref.py) on the CPU: it equals the backward
kernels executed on the host (tests/emu, g++ -ffp-contract=off) bit for bit, stays near the oracle's float64 autograd, is exact
on integer data, routes hand-built ties to the first slot across chunk boundaries, and its fma is correctly rounded."""
import ctypes as C
import importlib.util
import os
import shutil
from fractions import Fraction

import numpy as np
import pytest
import torch

import backward_paths_ref as B
import forward_paths_ref as FR
from oracle import pna_oracle as O
from pna_b200 import _lib

AGGRS = ["sum", "mean", "min", "max", "var", "std"]
SCALERS = ["identity", "linear", "inverse_linear"]        # no logarithm: host and kernel factors are the same IEEE divisions
AVG = {"log": 1.7, "lin": 4.3}
SPLIT, CHUNK = 16, 4

needs_gxx = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")


@pytest.fixture(scope="module")
def emu():
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(here, "emu", "build_emu.py"))
    build_emu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build_emu)
    try:
        L = C.CDLL(build_emu.build("pna_aggregate_bwd.cu"))
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    A = C.POINTER(_lib.AggStruct)
    L.emu_last_error.restype = C.c_char_p
    L.pna_aggregate_bwd.argtypes = [A, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    L.pna_aggregate_bwd_coef.argtypes = [A, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32, C.c_void_p, C.c_int64,
                                         C.c_void_p, C.c_int64, C.c_void_p]
    L.pna_aggregate_bwd_slots.argtypes = [A, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p,
                                          C.c_int64, C.c_void_p]
    return L


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def graph(seed, n=90, e=900, fixed=None):
    """random edges into rows >= 10, rows 0..9 fixed degrees around the split threshold and chunk multiples, the last rows
    isolated"""
    rng = np.random.default_rng(seed)
    fixed = fixed or {0: SPLIT - 1, 1: SPLIT, 2: 6 * CHUNK, 3: 6 * CHUNK + 1, 4: 61}
    dst = np.concatenate([rng.integers(10, n - 4, e)] + [np.full(d, r) for r, d in fixed.items()])
    src = rng.integers(0, n, dst.size)
    p = rng.permutation(dst.size)
    return src[p], dst[p], n


class Case:
    """One backward call on host data: CSR, inputs (fp32 values of the dtype), descriptor pieces."""

    def __init__(self, src, dst, n, f, dtype, seed, bias=False, towers=1, has_self=False, aggrs=AGGRS, scalers=SCALERS,
                 relu_var=False, ints=None):
        self.rowptr, self.col, self.info, self.items = FR.host_csr(src, dst, n, SPLIT, CHUNK)
        self.n, self.f, self.dtype, self.towers, self.has_self = n, f, dtype, towers, has_self
        self.aggrs, self.scalers, self.relu_var = list(aggrs), list(scalers), relu_var
        g = torch.Generator().manual_seed(seed)
        rnd = (lambda *s: torch.randint(-ints, ints + 1, s, generator=g).float()) if ints else (lambda *s: torch.randn(*s, generator=g))
        self.x = rnd(n, f).to(dtype)
        self.bias = rnd(n, f).to(dtype) if bias else None
        ft = f // towers
        self.width = towers * (int(has_self) + len(aggrs) * len(scalers)) * ft
        self.go = rnd(n, self.width).to(dtype)
        self.deg = np.diff(self.rowptr)

    def np(self, t):
        return None if t is None else t.float().numpy()

    def descriptor(self, scratch):
        self._keep = [torch.from_numpy(self.rowptr.astype(np.int32)), torch.from_numpy(self.col.astype(np.int32)),
                      torch.from_numpy(self.info.astype(np.int32).reshape(-1)), torch.from_numpy(self.items.astype(np.int32).reshape(-1))]
        rp, col, info, items = self._keep
        na, ac = _lib.pack_codes(self.aggrs, _lib.AGGR_CODES, "aggregator")
        ns, sc = _lib.pack_codes(self.scalers, _lib.SCALER_CODES, "scaler")
        return _lib.AggStruct(
            gathered=self.x.data_ptr(), ld_gathered=self.f, rowptr=rp.data_ptr(), col=col.data_ptr(),
            row_bias=None if self.bias is None else self.bias.data_ptr(), ld_row_bias=self.f,
            self_feat=1 if self.has_self else None, n_rows=self.n, n_feat=self.f, n_towers=self.towers,
            dtype=_lib.PNA_F32 if self.dtype == torch.float32 else _lib.PNA_BF16, n_aggr=na, aggr_codes=ac, n_scalers=ns,
            scaler_codes=sc, avg_log=AVG["log"], avg_lin=AVG["lin"], flags=_lib.FLAG_RELU_VAR if self.relu_var else 0,
            split_threshold=SPLIT, chunk_edges=CHUNK, hub_info=info.data_ptr() if len(self.info) else None,
            chunk_items=items.data_ptr() if len(self.items) else None, n_hubs=len(self.info), n_chunks=len(self.items),
            hub_partials=scratch.data_ptr())

    def reference(self):
        x, bias = self.np(self.x), self.np(self.bias)
        st = B.row_stats_bwd(x, self.rowptr, self.col, self.info, CHUNK, bias)
        scales = FR.host_scales(self.deg, self.scalers, AVG["log"], AVG["lin"])
        c = B.coefficients(st, self.deg, self.np(self.go), scales, self.aggrs, towers=self.towers, has_self=self.has_self,
                           relu_var=self.relu_var)
        gm, gb, shares = B.slot_grads(c, st, x, self.rowptr, self.col, self.info, CHUNK, bias)
        return st, c, gm, gb, shares

    def scratch(self):
        return torch.zeros(((len(self.items) + len(self.info)) * 6 + 1, self.f))


def run_slots(emu, cs):
    scratch = cs.scratch()
    d = cs.descriptor(scratch)
    E = len(cs.col)
    gs = torch.full((E, cs.f), float("nan"))
    gb = torch.full((cs.n, cs.f), float("nan"))
    rc = emu.pna_aggregate_bwd_slots(C.byref(d), cs.go.data_ptr(), cs.width, 0, cs.f, gs.data_ptr(), cs.f, gb.data_ptr(), cs.f, None)
    assert rc == 0, emu.emu_last_error()
    return gs.numpy(), gb.numpy()


def run_coef(emu, cs):
    scratch = cs.scratch()
    d = cs.descriptor(scratch)
    fp = (cs.f + 3) // 4 * 4
    coef = torch.full((cs.n, 2 * fp), float("nan"))
    gg = torch.zeros(cs.n, cs.f)
    gb = torch.full((cs.n, cs.f), float("nan"))
    rc = emu.pna_aggregate_bwd_coef(C.byref(d), cs.go.data_ptr(), cs.width, coef.data_ptr(), 2 * fp, fp, gg.data_ptr(), cs.f,
                                    gb.data_ptr(), cs.f, None)
    assert rc == 0, emu.emu_last_error()
    return coef.numpy()[:, :cs.f], coef.numpy()[:, fp:fp + cs.f], gg.numpy(), gb.numpy()


EMU_CASES = [
    # F, dtype, bias, towers, self_feat, options
    (12, torch.float32, False, 1, False, {}),
    (12, torch.float32, True, 1, False, {}),
    (16, torch.bfloat16, False, 1, False, {}),
    (16, torch.bfloat16, True, 1, False, {}),
    (16, torch.float32, True, 2, True, {}),
    (32, torch.bfloat16, True, 2, True, {}),
    (7, torch.float32, True, 1, False, {"relu_var": True}),
    (12, torch.float32, False, 1, False, {"aggrs": ["var", "_skip", "max", "sum", "_skip", "std"]}),
]


@needs_gxx
@pytest.mark.parametrize("f,dtype,bias,towers,has_self,opt", EMU_CASES)
def test_restatement_equals_emulated_kernels(emu, f, dtype, bias, towers, has_self, opt):
    src, dst, n = graph(f + 3 * towers)
    cs = Case(src, dst, n, f, dtype, seed=f, bias=bias, towers=towers, has_self=has_self, **opt)
    assert {1, 2, 3, 4} <= set(cs.info[:, 0].tolist()) and 0 not in cs.info[:, 0] and (cs.info[:, 2] > 1).all()
    st, c, gm, gb, _ = cs.reference()
    gs, gb_s = run_slots(emu, cs)
    assert np.array_equal(bits(gs), bits(gm))
    assert np.array_equal(bits(gb_s), bits(gb))
    c0p, c1, gg, gb_c = run_coef(emu, cs)
    want0, want1, want_gb = B.coef_rows(c, st, cs.deg, cs.np(cs.bias))
    has_in = cs.deg > 0
    assert (~has_in).any() and np.isnan(c0p[~has_in]).all()       # rows without in-edges: never written, never read
    assert np.array_equal(bits(c0p[has_in]), bits(want0[has_in]))
    assert np.array_equal(bits(c1[has_in]), bits(want1[has_in]))
    assert np.array_equal(bits(gb_c[has_in]), bits(want_gb[has_in]))
    assert np.array_equal(gb_c[~has_in], np.zeros_like(gb_c[~has_in]))
    r, fcol, v = B.routed_terms(c, st, cs.deg, cs.col)
    terms = np.zeros((len(v), f), np.float32)
    terms[np.arange(len(v)), fcol] = v
    s, bound = B.order_free_sum(n, r, terms)
    assert B.within_order_free(gg, s, bound).all()
    if "min" in cs.aggrs or "max" in cs.aggrs:
        assert len(v) > 0


def test_restatement_is_near_the_float64_autograd():
    """Bar from the term magnitudes: every per-slot gradient is a handful of fp32 operations on coefficients that each sum
    S scaled terms and divide by statistics over deg slots; allow 8 (deg_max + S + 4) u of sum |c0| + |c1 m| + |gmin| + |gmax|
    over the slots of each source (u = 2^-24)."""
    src, dst, n = graph(1)
    cs = Case(src, dst, n, 10, torch.float32, seed=2, bias=True)
    st, c, gm, gb, _ = cs.reference()
    x, bias = cs.np(cs.x), cs.np(cs.bias)
    row = B.slot_rows(cs.rowptr)
    got = np.zeros((n, 10), np.float64)
    np.add.at(got, cs.col, gm.astype(np.float64))
    # the oracle's autograd in float64
    xr = torch.from_numpy(x).double().requires_grad_(True)
    br = torch.from_numpy(bias).double().requires_grad_(True)
    ei_dst = torch.from_numpy(row)
    msg = xr[torch.from_numpy(cs.col)] + br[ei_dst]
    out = O.pyg_aggregate(msg, ei_dst, n, AGGRS, SCALERS, AVG)
    (out * torch.from_numpy(cs.np(cs.go)).double()).sum().backward()
    m = x[cs.col] + bias[row]
    mag = np.abs(c[0][row]) + np.abs(c[1][row] * m) + np.abs(c[2][row]) + np.abs(c[3][row])
    a = np.zeros((n, 10))
    np.add.at(a, cs.col, mag)
    bar = 8 * (int(cs.deg.max()) + len(SCALERS) + 4) * 2.0 ** -24 * a
    assert (np.abs(got - xr.grad.numpy()) <= bar).all()
    ab = np.zeros((n, 10))
    np.add.at(ab, row, mag)
    assert (np.abs(gb - br.grad.numpy()) <= 8 * (int(cs.deg.max()) + len(SCALERS) + 4) * 2.0 ** -24 * ab).all()


def test_integer_data_is_exact_in_every_order():
    """Integer features and upstream gradients, sum / min / max with the identity scaler: every per-slot gradient and every
    partial sum is an integer below 2^24, so every summation order gives the float64 value."""
    src, dst, n = graph(3)
    cs = Case(src, dst, n, 8, torch.float32, seed=4, aggrs=["sum", "min", "max"], scalers=["identity"], ints=3)
    st, c, gm, gb, shares = cs.reference()
    row = B.slot_rows(cs.rowptr)
    s, bound = B.order_free_sum(n, cs.col, gm)
    want = np.zeros((n, 8))
    np.add.at(want, cs.col, gm.astype(np.float64))
    assert np.array_equal(s, want)
    for order in (np.arange(len(row)), np.random.default_rng(5).permutation(len(row))):
        acc = np.zeros((n, 8), np.float32)
        for k in order:
            acc[cs.col[k]] = acc[cs.col[k]] + gm[k]
        assert np.array_equal(acc.astype(np.float64), want)
    gb64 = np.zeros((n, 8))
    np.add.at(gb64, row, gm.astype(np.float64))
    assert np.array_equal(gb.astype(np.float64), gb64)
    # the closed form of the coefficient mode equals it too (rows with in-edges: the kernels write 0 for the others)
    has_in = cs.deg > 0
    assert np.array_equal(B.coef_rows(c, st, cs.deg)[2][has_in].astype(np.float64), gb64[has_in])
    # and the statistics are float64's
    exact = FR.stats_f64(cs.np(cs.x), cs.rowptr, cs.col)
    for k in range(4):
        assert np.array_equal(st[k].astype(np.float64), exact[:, k])


# one split row of 12 slots in chunks of 4 (split threshold 4): feature 0's minimum -5 first at slot 5 (chunk 1), again at slot 6
# (same chunk) and slot 9 (chunk 2); its maximum 7 at slots 2 and 11.  Feature 1's minimum at slot 3, the last of chunk 0, and
# at slots 4 (first of chunk 1) and 8 (first of chunk 2); its maximum 9 at slots 5 and 7.
TIE_VALUES = np.array([
    [0, 1], [1, 2], [7, 3], [2, -4],
    [3, -4], [-5, 9], [-5, 0], [4, 9],
    [5, -4], [-5, 1], [6, 2], [7, 3]], np.float32)
TIE_ARGS = {"amn": [5, 3], "amx": [2, 5]}


@needs_gxx
def test_hand_built_ties_route_to_the_first_slot(emu):
    n = 14
    src = np.arange(1, 13)                      # slot k of row 0 gathers row k + 1
    dst = np.zeros(12, np.int64)
    x = np.zeros((n, 2), np.float32)
    x[1:13] = TIE_VALUES
    rowptr, col, info, items = FR.host_csr(src, dst, n, 4, 4)
    assert info.tolist() == [[0, 0, 3, 12]]
    st = B.row_stats_bwd(x, rowptr, col, info, 4)
    assert st[4][0].tolist() == TIE_ARGS["amn"] and st[5][0].tolist() == TIE_ARGS["amx"]
    light = B.row_stats_bwd(x, rowptr, col, np.zeros((0, 4), np.int64), 4)     # one pass over the row: the same slots
    assert light[4][0].tolist() == TIE_ARGS["amn"] and light[5][0].tolist() == TIE_ARGS["amx"]
    # the emulated kernels: grad_out = 1 for min and max, so grad_m is 1 exactly at each arg slot
    L = emu
    rp, cl = torch.from_numpy(rowptr.astype(np.int32)), torch.from_numpy(col.astype(np.int32))
    inf, it = torch.from_numpy(info.astype(np.int32).reshape(-1)), torch.from_numpy(items.astype(np.int32).reshape(-1))
    xt = torch.from_numpy(x)
    scratch = torch.zeros((len(items) + 1) * 6, 2)
    na, ac = _lib.pack_codes(["min", "max"], _lib.AGGR_CODES, "aggregator")
    ns, sc = _lib.pack_codes(["identity"], _lib.SCALER_CODES, "scaler")
    d = _lib.AggStruct(gathered=xt.data_ptr(), ld_gathered=2, rowptr=rp.data_ptr(), col=cl.data_ptr(), n_rows=n, n_feat=2,
                       n_towers=1, dtype=_lib.PNA_F32, n_aggr=na, aggr_codes=ac, n_scalers=ns, scaler_codes=sc, avg_log=1.0,
                       avg_lin=1.0, split_threshold=4, chunk_edges=4, hub_info=inf.data_ptr(), chunk_items=it.data_ptr(),
                       n_hubs=1, n_chunks=3, hub_partials=scratch.data_ptr())
    go = torch.tensor([[1.0, 0.0, 0.0, 0.0]] + [[0.0] * 4] * (n - 1))          # columns: min f0, min f1, max f0, max f1
    gs = torch.full((12, 2), float("nan"))
    assert L.pna_aggregate_bwd_slots(C.byref(d), go.data_ptr(), 4, 0, 2, gs.data_ptr(), 2, None, 0, None) == 0
    want = np.zeros((12, 2), np.float32)
    want[TIE_ARGS["amn"][0], 0] = 1
    assert np.array_equal(gs.numpy(), want)
    go = torch.zeros(n, 4)
    go[0] = torch.tensor([0.0, 1.0, 2.0, 4.0])
    gs = torch.full((12, 2), float("nan"))
    assert L.pna_aggregate_bwd_slots(C.byref(d), go.data_ptr(), 4, 0, 2, gs.data_ptr(), 2, None, 0, None) == 0
    want = np.zeros((12, 2), np.float32)
    want[TIE_ARGS["amn"][1], 1] += 1
    want[TIE_ARGS["amx"][0], 0] += 2
    want[TIE_ARGS["amx"][1], 1] += 4
    assert np.array_equal(gs.numpy(), want)


def _round_fraction_to_f32(q: Fraction) -> np.float32:
    """nearest float32 of an exact rational, ties to even"""
    f = np.float32(float(q))
    cands = [f, np.nextafter(f, np.float32(np.inf)), np.nextafter(f, np.float32(-np.inf))]
    dist = [(abs(Fraction(float(c)) - q), int(np.array(c).view(np.uint32)) & 1, c) for c in cands if np.isfinite(c)]
    dist.sort(key=lambda t: (t[0], t[1]))
    return dist[0][2]


def test_fma32_is_correctly_rounded():
    rng = np.random.default_rng(11)
    a = (rng.standard_normal(3000) * np.exp2(rng.integers(-20, 20, 3000))).astype(np.float32)
    b = (rng.standard_normal(3000) * np.exp2(rng.integers(-20, 20, 3000))).astype(np.float32)
    c = (rng.standard_normal(3000) * np.exp2(rng.integers(-40, 40, 3000))).astype(np.float32)
    # halfway cases: c puts a*b + c exactly on (or one fp32 step of c beside) the midpoint of two floats of a*b's binade
    p = a.astype(np.float64) * b.astype(np.float64)
    r = p.astype(np.float32)
    half = (np.nextafter(r, np.float32(np.inf)).astype(np.float64) - r.astype(np.float64)) / 2
    mid = (r.astype(np.float64) + half) - p
    ok = mid.astype(np.float32).astype(np.float64) == mid
    c_mid = mid[ok].astype(np.float32)
    A = np.concatenate([a, a[ok], a[ok], a[ok]])
    Bv = np.concatenate([b, b[ok], b[ok], b[ok]])
    Cv = np.concatenate([c, c_mid, np.nextafter(c_mid, np.float32(np.inf)), np.nextafter(c_mid, np.float32(-np.inf))])
    assert ok.sum() > 1000
    got = B.fma32(A, Bv, Cv)
    want = np.array([_round_fraction_to_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(A, Bv, Cv)], np.float32)
    assert np.array_equal(bits(got), bits(want))
    # where float64 a*b + c double-rounds, the helper must differ from it
    naive = (A.astype(np.float64) * Bv.astype(np.float64) + Cv.astype(np.float64)).astype(np.float32)
    assert (bits(naive) != bits(want)).any()


def test_order_free_bound_holds_for_shuffled_fp32_sums():
    rng = np.random.default_rng(12)
    rows = rng.integers(0, 20, 2000)
    terms = (rng.standard_normal((2000, 3)) * np.exp2(rng.integers(-8, 8, (2000, 1)))).astype(np.float32)
    s, bound = B.order_free_sum(20, rows, terms)
    for seed in range(3):
        acc = np.zeros((20, 3), np.float32)
        for k in np.random.default_rng(seed).permutation(2000):
            acc[rows[k]] = acc[rows[k]] + terms[k]
        assert B.within_order_free(acc, s, bound).all()
    assert not B.within_order_free(acc * np.float32(1 + 1e-3), s, bound).all()


def test_bwd_instance_restates_the_launcher():
    assert B.bwd_instance(4, 4, True) == (4, 1, 1)
    assert B.bwd_instance(8, 4, True) == (4, 2, 1)
    assert B.bwd_instance(64, 4, True) == (4, 16, 1)
    assert B.bwd_instance(128, 4, True) == (4, 32, 1)
    assert B.bwd_instance(256, 4, True) == (4, 32, 2)
    assert B.bwd_instance(1024, 4, True) == (4, 32, 8)
    assert B.bwd_instance(75, 4, False) == (1, 32, 3)
    assert B.bwd_instance(3, 4, False) == (1, 4, 1)
    assert B.bwd_instance(8, 2, True) == (8, 1, 1)
    assert B.bwd_instance(512, 2, True) == (8, 32, 2)
    assert B.bwd_instance(64, 4, True)[2] == 1 and B.bwd_instance(72, 4, True) == (4, 32, 1)
    assert B.bwd_vec_ok(16, 4, [(256, 16), (512, 48)])
    assert not B.bwd_vec_ok(25, 4, [(256, 100)])                 # Ft = 25
    assert not B.bwd_vec_ok(16, 4, [(256, 16), (516, 48)])       # misaligned base
    assert not B.bwd_vec_ok(16, 4, [(256, 18)])                  # odd pitch
    assert B.bwd_vec_ok(8, 2, [(0, 8)]) and not B.bwd_vec_ok(8, 2, [(0, 12)])
