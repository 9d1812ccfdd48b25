"""The deterministic backward (pna_aggregate_bwd_slots, csrc/pna_aggregate_bwd.cu) executed on the HOST, thread by thread
(tests/emu): its per-slot gradients are the atomic path's per-edge values bit for bit, its feature slabs are column slices
of the full-width run, summing them per source row in ascending slot order gives the atomic backward's result, and the
split-row grad_row_bias adds the chunks' slot-order sums in chunk order.  Step 2 on the GPU (the forward kernel over the
slot-transposed CSR) is covered by tests/test_gpu_bwd_deterministic.py."""
import ctypes as C
import shutil

import numpy as np
import pytest
import torch

from oracle import pna_oracle as O
from pna_b200 import _lib

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

AGGRS = ["sum", "mean", "min", "max", "var", "std"]
SCALERS = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]
SPLIT, CHUNK = 16, 8


@pytest.fixture(scope="module")
def emu():
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "build_emu.py"))
    build_emu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build_emu)
    try:
        L = C.CDLL(build_emu.build("pna_aggregate_bwd.cu"))
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    L.pna_aggregate_bwd.argtypes = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    L.pna_aggregate_bwd_slots.argtypes = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                          C.c_void_p, C.c_int64, C.c_void_p]
    return L


def host_csr(src, dst, n):
    """Destination-sorted CSR (stable in edge order) + the split-row tables, as pna_csr_build lays them out."""
    order = torch.sort(dst, stable=True).indices
    col = src[order].to(torch.int32).contiguous()
    deg = torch.bincount(dst, minlength=n)
    rowptr = torch.zeros(n + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).to(torch.int32)
    hubs, chunks = [], []
    for r in (deg >= SPLIT).nonzero().flatten().tolist():
        nch = (int(deg[r]) + CHUNK - 1) // CHUNK
        hubs.append([r, len(chunks), nch, int(deg[r])])
        chunks += [[len(hubs) - 1, j] for j in range(nch)]
    hub_info = torch.tensor(hubs, dtype=torch.int32).reshape(-1, 4).contiguous()
    chunk_items = torch.tensor(chunks, dtype=torch.int32).reshape(-1, 2).contiguous()
    return rowptr, col, hub_info, chunk_items


class Case:
    """One graph + inputs, and the host-emulated entry points on it."""

    def __init__(self, emu, src, dst, n, x, bias, w, aggrs, scalers, towers=1, relu_var=False):
        self.emu, self.n, self.x, self.bias, self.towers = emu, n, x, bias, towers
        self.src, self.dst, self.aggrs, self.scalers, self.relu_var = src, dst, aggrs, scalers, relu_var
        self.rowptr, self.col, self.hub_info, self.chunk_items = host_csr(src, dst, n)
        self.E, self.F = self.col.numel(), x.size(1)
        self.avg = O.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
        self.w = w.to(x.dtype).contiguous()

    def desc(self, x, col):
        na, ac = _lib.pack_codes(self.aggrs, _lib.AGGR_CODES, "aggregator")
        ns, sc = _lib.pack_codes(self.scalers, _lib.SCALER_CODES, "scaler")
        self.scratch = torch.full(((self.chunk_items.size(0) + self.hub_info.size(0)) * 6, self.F), float("nan"))
        b = self.bias
        return _lib.AggStruct(
            gathered=x.data_ptr(), ld_gathered=x.stride(0), rowptr=self.rowptr.data_ptr(), col=None if col is None else col.data_ptr(),
            row_bias=None if b is None else b.data_ptr(), ld_row_bias=0 if b is None else b.stride(0),
            n_rows=self.n, n_feat=self.F, n_towers=self.towers, dtype=_lib.PNA_F32 if x.dtype == torch.float32 else _lib.PNA_BF16,
            n_aggr=na, aggr_codes=ac, n_scalers=ns, scaler_codes=sc, avg_log=float(self.avg["log"]), avg_lin=float(self.avg["lin"]),
            flags=_lib.FLAG_RELU_VAR if self.relu_var else 0, split_threshold=SPLIT, chunk_edges=CHUNK,
            hub_info=self.hub_info.data_ptr() if self.hub_info.numel() else None,
            chunk_items=self.chunk_items.data_ptr() if self.chunk_items.numel() else None,
            n_hubs=self.hub_info.size(0), n_chunks=self.chunk_items.size(0),
            hub_partials=self.scratch.data_ptr() if self.scratch.numel() else None)

    def slots(self, f0=0, fc=None):
        """pna_aggregate_bwd_slots (gathered rows through col): grad_slots [E, fc], grad_row_bias [N, F] (slab columns)."""
        fc = self.F - f0 if fc is None else fc
        d = self.desc(self.x, self.col)
        gs = torch.full((self.E, fc), float("nan"))
        gb = torch.full((self.n, self.F), float("nan"))
        rc = self.emu.pna_aggregate_bwd_slots(C.byref(d), self.w.data_ptr(), self.w.stride(0), f0, fc, gs.data_ptr(), fc,
                                              gb.data_ptr(), self.F, None)
        assert rc == 0, self.emu.emu_last_error()
        return gs, gb

    def atomic(self, materialised=False):
        """pna_aggregate_bwd: through col, or (materialised) on x[col] in CSR order with col == NULL (per-slot gradients)."""
        x = self.x[self.col.long()].contiguous() if materialised else self.x
        d = self.desc(x, None if materialised else self.col)
        gg = torch.zeros(x.size(0), self.F)
        gb = torch.full((self.n, self.F), float("nan"))
        rc = self.emu.pna_aggregate_bwd(C.byref(d), self.w.data_ptr(), self.w.stride(0), gg.data_ptr(), self.F, gb.data_ptr(),
                                        self.F, None)
        assert rc == 0, self.emu.emu_last_error()
        return gg, gb

    def source_sums(self, gs):
        """Sequential fp32 sum of grad_slots over every source row's slots, in ascending slot order."""
        acc = np.zeros((self.x.size(0), gs.size(1)), dtype=np.float32)
        g, col = gs.numpy(), self.col.numpy()
        for s in range(self.E):
            acc[col[s]] = acc[col[s]] + g[s]
        return torch.from_numpy(acc)

    def chunk_ordered_bias(self, gs):
        """grad_row_bias restated: rows below the threshold add their slots in order; split rows add each chunk's slot-order
        sum, chunks in order."""
        g, rp = gs.numpy(), self.rowptr.numpy()
        out = np.zeros((self.n, gs.size(1)), dtype=np.float32)
        for r in range(self.n):
            beg, end = int(rp[r]), int(rp[r + 1])
            if end - beg >= SPLIT:
                for c0 in range(beg, end, CHUNK):
                    part = np.zeros(gs.size(1), dtype=np.float32)
                    for s in range(c0, min(c0 + CHUNK, end)):
                        part = part + g[s]
                    out[r] = out[r] + part
            else:
                for s in range(beg, end):
                    out[r] = out[r] + g[s]
        return torch.from_numpy(out)

    def oracle(self):
        """The reference's autograd (PyG flavour, fp32): x_j + row_bias_i per message, per tower."""
        assert not self.relu_var
        xr = self.x.float().clone().requires_grad_(True)
        br = self.bias.float().clone().requires_grad_(True) if self.bias is not None else None
        msg = xr[self.src] + (br[self.dst] if br is not None else 0.0)
        ft = self.F // self.towers
        outs = [O.pyg_aggregate(msg[:, t * ft:(t + 1) * ft], self.dst, self.n, self.aggrs, self.scalers, self.avg)
                for t in range(self.towers)]
        (torch.cat(outs, 1) * self.w.float()).sum().backward()
        return xr.grad, None if br is None else br.grad


def graph(n, e, seed, big=0, hot_src=0):
    """Random multigraph; `big` slots go to one row (split: several chunks) and SPLIT more to another (exactly at the threshold);
    `hot_src` edges leave one source row."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, n - 5, (e,), generator=g)          # the last rows are isolated
    if big:
        dst[:big] = 2
        dst[big:big + SPLIT] = 7
    if hot_src:
        src[-hot_src:] = 3
    return src, dst, g


def make(emu, f, towers=1, with_bias=True, dtype=torch.float32, aggrs=AGGRS, scalers=SCALERS, relu_var=False, n=60, e=420,
         big=70, seed=0, hot_src=0):
    src, dst, g = graph(n, e, seed + f, big=big, hot_src=hot_src)
    x = torch.randn(n, f, generator=g).to(dtype)
    bias = torch.randn(n, f, generator=g).to(dtype) if with_bias else None
    w = torch.randn(n, len(aggrs) * len(scalers) * f, generator=g)
    return Case(emu, src, dst, n, x, bias, w, aggrs, scalers, towers, relu_var)


CASES = [   # f, towers, bias, dtype, relu_var
    (12, 1, True, torch.float32, False), (12, 1, False, torch.float32, True), (10, 1, True, torch.float32, False),
    (16, 2, True, torch.float32, True), (40, 1, False, torch.float32, False), (3, 1, True, torch.float32, False),
    (160, 1, True, torch.float32, False), (192, 4, True, torch.float32, True), (16, 1, True, torch.bfloat16, False),
    (24, 3, True, torch.bfloat16, True), (10, 1, True, torch.bfloat16, False),
]


@pytest.mark.parametrize("f,towers,with_bias,dtype,relu_var", CASES)
def test_slots_are_the_per_slot_gradient_of_the_materialised_messages(emu, f, towers, with_bias, dtype, relu_var):
    """grad_slots (through col) == pna_aggregate_bwd's per-slot gradient with col == NULL on x[col], bit for bit; split rows
    included, so grad_row_bias (slot order, chunks in order) equals what the sequential atomics add."""
    c = make(emu, f, towers, with_bias, dtype, relu_var=relu_var)
    assert c.hub_info.size(0) == 2
    gs, gb = c.slots()
    want, want_b = c.atomic(materialised=True)
    assert torch.equal(gs, want)
    if with_bias:
        assert torch.equal(gb, want_b)
    assert torch.isfinite(gs).all()


@pytest.mark.parametrize("f,towers,with_bias,dtype,relu_var", CASES)
def test_every_feature_slab_is_a_column_slice_of_the_full_width_run(emu, f, towers, with_bias, dtype, relu_var):
    c = make(emu, f, towers, with_bias, dtype, relu_var=relu_var, seed=5)
    gs, gb = c.slots()
    al = 4 if dtype == torch.float32 else 8
    for width in sorted({al, 2 * al, 3 * al}):
        for f0 in range(0, f, width):
            fc = min(width, f - f0)
            gs_s, gb_s = c.slots(f0, fc)
            assert torch.equal(gs_s, gs[:, f0:f0 + fc]), (width, f0)
            if with_bias:
                assert torch.equal(gb_s[:, f0:f0 + fc], gb[:, f0:f0 + fc]), (width, f0)
                assert torch.isnan(gb_s[:, :f0]).all() and torch.isnan(gb_s[:, f0 + fc:]).all()   # other columns untouched


@pytest.mark.parametrize("f,towers,with_bias,dtype,relu_var", CASES)
def test_ordered_source_sums_equal_the_atomic_backward_without_split_rows(emu, f, towers, with_bias, dtype, relu_var):
    """No split rows in either direction: the emulated atomics add each source's slots in ascending slot order, so the
    sequential sum of grad_slots (what the forward kernel computes over the slot-transposed CSR) is the same bits."""
    c = make(emu, f, towers, with_bias, dtype, relu_var=relu_var, n=70, e=300, big=0, seed=9)
    assert c.hub_info.numel() == 0 and int(torch.bincount(c.src).max()) < SPLIT
    gs, gb = c.slots()
    gg, gb_atomic = c.atomic()
    assert torch.equal(c.source_sums(gs), gg)
    if with_bias:
        assert torch.equal(gb, gb_atomic)


@pytest.mark.parametrize("f,towers,with_bias,dtype", [(12, 1, True, torch.float32), (16, 2, True, torch.float32),
                                                      (160, 1, True, torch.float32), (24, 3, True, torch.bfloat16),
                                                      (10, 1, True, torch.float32), (40, 1, False, torch.float32)])
def test_split_row_bias_is_the_chunk_ordered_sum_and_matches_the_oracle(emu, f, towers, with_bias, dtype):
    # bf16 inputs tie often, and the oracle's min / max may route a tie elsewhere (tie routing: tests/test_bwd_emulated.py)
    aggrs = AGGRS if dtype == torch.float32 else ["mean", "std", "sum", "var"]
    c = make(emu, f, towers, with_bias, dtype, aggrs=aggrs, seed=11, big=90, hot_src=40)
    gs, gb = c.slots()
    want_x, want_b = c.oracle()
    # std has a slope of up to 158 at var ~ 0 and the sums run in fp32: the bar of tests/test_bwd_emulated.py
    tol = dict(rtol=1e-3, atol=5e-4) if dtype == torch.float32 else dict(rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(c.source_sums(gs), want_x.float(), **tol)
    if with_bias:
        assert torch.equal(gb, c.chunk_ordered_bias(gs))
        has_in = torch.bincount(c.dst, minlength=c.n) > 0
        torch.testing.assert_close(gb[has_in], want_b.float()[has_in], rtol=1e-3, atol=2e-3)
        assert torch.equal(gb[~has_in], torch.zeros_like(gb[~has_in]))


def test_every_aggregator_and_scaler_subset(emu):
    """Random widths, towers, aggregator / scaler subsets, row_bias on and off, relu_var, graphs with and without split rows:
    every launch geometry of the per-slot variant, each against the per-slot gradient of the materialised messages."""
    import random
    rnd = random.Random(1)
    for it in range(40):
        towers = rnd.choice([1, 1, 2, 3])
        f = rnd.choice([1, 2, 4, 5, 8, 12, 16, 33]) * towers
        aggrs, scalers = rnd.sample(AGGRS, rnd.randint(1, 6)), rnd.sample(SCALERS, rnd.randint(1, 5))
        dtype = rnd.choice([torch.float32, torch.float32, torch.bfloat16])
        n, e = rnd.randint(8, 60), rnd.randint(1, 400)
        c = make(emu, f, towers, rnd.random() < 0.5, dtype, aggrs, scalers, relu_var=rnd.random() < 0.3, n=n, e=e,
                 big=rnd.choice([0, 0, min(e - SPLIT, 60)]) if e > 2 * SPLIT else 0, seed=100 + it)
        gs, gb = c.slots()
        want, want_b = c.atomic(materialised=True)
        what = f"case {it}: F={f} towers={towers} {dtype} {aggrs} {scalers}"
        assert torch.equal(gs, want), what
        if c.bias is not None:
            assert torch.equal(gb, want_b), what


PNA_ERR_BAD_ARG, PNA_ERR_UNSUPPORTED = -1, -2      # include/pna_b200.h


def test_bad_slabs_and_peer_descriptors_are_refused(emu):
    c = make(emu, 12, seed=3)
    d = c.desc(c.x, c.col)
    gs = torch.zeros(c.E, 12)
    # unaligned start, empty, past n_feat, unaligned end inside the row, negative start
    for f0, fc in [(2, 4), (0, 0), (0, 13), (8, 8), (-4, 4), (0, 6)]:
        rc = emu.pna_aggregate_bwd_slots(C.byref(d), c.w.data_ptr(), c.w.stride(0), f0, fc, gs.data_ptr(), 12, None, 0, None)
        assert rc == PNA_ERR_BAD_ARG, (f0, fc, rc)
    rc = emu.pna_aggregate_bwd_slots(C.byref(d), c.w.data_ptr(), c.w.stride(0), 0, 12, gs.data_ptr(), 8, None, 0, None)
    assert rc == PNA_ERR_BAD_ARG                                          # ld_grad_slots < f_count
    rc = emu.pna_aggregate_bwd_slots(C.byref(d), c.w.data_ptr(), c.w.stride(0), 0, 12, None, 12, None, 0, None)
    assert rc == PNA_ERR_BAD_ARG                                          # no grad_slots
    d.peer_gathered = 256                                                 # never dereferenced: refused first
    rc = emu.pna_aggregate_bwd_slots(C.byref(d), c.w.data_ptr(), c.w.stride(0), 0, 12, gs.data_ptr(), 12, None, 0, None)
    assert rc == PNA_ERR_UNSUPPORTED
    assert torch.equal(gs, torch.zeros_like(gs))
