"""The peer plane's backward on the HOST (tests/emu): pna_aggregate_bwd_peer_slots executed thread by thread for W "ranks"
whose feature rows are separate host buffers named by a pointer table, col = owner << shift | row.  Every rank's per-slot
gradients and grad_row_bias must be what pna_aggregate_bwd_slots stores for the same slots of the unpartitioned graph, bit
for bit; the owners' return (pna_halo_grad_pull on the reverse slot plan) must be the sequential fp32 sum of every source
row's slots in ascending slot order of the whole graph.  The GPU run is tests/test_gpu_peer_grad.py."""
import ctypes as C
import importlib.util
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import pna_oracle as O
from pna_b200 import _lib, dist as pd

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

AGGRS = ["mean", "max", "min", "std", "sum", "var"]
SCALERS = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]
SPLIT, CHUNK = 16, 8
PNA_ERR_BAD_ARG, PNA_ERR_UNSUPPORTED = -1, -2      # include/pna_b200.h


def _build(name):
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "build_emu.py"))
    build_emu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build_emu)
    try:
        L = C.CDLL(build_emu.build(name))
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    return L


@pytest.fixture(scope="module")
def emu():
    L = _build("pna_aggregate_bwd.cu")
    args = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
            C.c_void_p]
    L.pna_aggregate_bwd_slots.argtypes = args
    L.pna_aggregate_bwd_peer_slots.argtypes = args
    return L


@pytest.fixture(scope="module")
def emu_peer():
    L = _build("pna_peer.cu")
    L.pna_halo_grad_pull.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                     C.c_int64, C.c_int32, C.c_void_p]
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


class Graph:
    """One CSR (the whole graph, or one rank's rows) and its descriptor for the per-slot backward."""

    def __init__(self, src, dst, n, x, bias, w, avg, towers):
        self.n, self.x, self.bias, self.w, self.avg, self.towers = n, x, bias, w, avg, towers
        self.rowptr, self.col, self.hub_info, self.chunk_items = host_csr(src, dst, n)
        self.E, self.F = self.col.numel(), x.size(1)

    def desc(self, peer=None):
        na, ac = _lib.pack_codes(AGGRS, _lib.AGGR_CODES, "aggregator")
        ns, sc = _lib.pack_codes(SCALERS, _lib.SCALER_CODES, "scaler")
        self.scratch = torch.full(((self.chunk_items.size(0) + self.hub_info.size(0)) * 6, self.F), float("nan"))
        b = self.bias
        d = _lib.AggStruct(
            gathered=self.x.data_ptr(), ld_gathered=self.x.stride(0), rowptr=self.rowptr.data_ptr(),
            col=self.col.data_ptr() if self.E else None,
            row_bias=None if b is None else b.data_ptr(), ld_row_bias=0 if b is None else b.stride(0),
            n_rows=self.n, n_feat=self.F, n_towers=self.towers, dtype=_lib.PNA_F32 if self.x.dtype == torch.float32 else _lib.PNA_BF16,
            n_aggr=na, aggr_codes=ac, n_scalers=ns, scaler_codes=sc, avg_log=float(self.avg["log"]), avg_lin=float(self.avg["lin"]),
            split_threshold=SPLIT, chunk_edges=CHUNK,
            hub_info=self.hub_info.data_ptr() if self.hub_info.numel() else None,
            chunk_items=self.chunk_items.data_ptr() if self.chunk_items.numel() else None,
            n_hubs=self.hub_info.size(0), n_chunks=self.chunk_items.size(0),
            hub_partials=self.scratch.data_ptr() if self.scratch.numel() else None)
        if peer is not None:
            d.peer_gathered, d.peer_shift = peer
        return d

    def slots(self, fn, f0, fc, peer=None, gs=None):
        d = self.desc(peer)
        gs = torch.full((max(self.E, 1), fc), float("nan")) if gs is None else gs
        gb = torch.full((self.n, self.F), float("nan"))
        rc = fn(C.byref(d), self.w.data_ptr(), self.w.stride(0), f0, fc, gs.data_ptr(), gs.stride(0), gb.data_ptr(), self.F, None)
        return rc, gs, gb


def setup(f, world, dtype, with_bias, towers=1, n=90, e=700, big=80, seed=0, pad=0):
    """A random multigraph over n nodes cut into `world` destination ranges, a row with `big` extra in-edges (split), and
    the inputs; returns the whole graph and every rank's CSR over owner|row-encoded sources with its row buffer."""
    g = torch.Generator().manual_seed(seed + 31 * f + world)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, n - 4, (e,), generator=g)                   # the last rows are isolated
    if big:
        src = torch.cat([src, torch.randint(0, n, (big,), generator=g)])
        dst = torch.cat([dst, torch.full((big,), n // 2)])
        p = torch.randperm(src.numel(), generator=g)
        src, dst = src[p], dst[p]
    x = torch.randn(n, f, generator=g).to(dtype)
    bias = torch.randn(n, f, generator=g).to(dtype) if with_bias else None
    w = torch.randn(n, towers * len(AGGRS) * len(SCALERS) * (f // towers), generator=g).to(dtype)
    deg = torch.bincount(dst, minlength=n)
    avg = O.avg_deg_from_histogram(torch.bincount(deg))
    whole = Graph(src, dst, n, x, bias, w, avg, towers)
    bounds = pd.partition_bounds(deg, world)
    shift = pd.peer_shift_for(bounds)
    rows_max = int((bounds[1:] - bounds[:-1]).max())
    bufs = []
    for r in range(world):
        b = torch.full((rows_max, f + pad), -3.0, dtype=dtype)         # pitch f + pad on every rank
        b[: int(bounds[r + 1] - bounds[r]), :f] = x[int(bounds[r]):int(bounds[r + 1])]
        bufs.append(b)
    table = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64)
    ranks = []
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        mine = (dst >= lo) & (dst < hi)
        enc = pd.encode_peer_sources(src[mine], bounds, shift)
        gr = Graph(enc, dst[mine] - lo, hi - lo, bufs[r][:, :f], None if bias is None else bias[lo:hi].contiguous(),
                   w[lo:hi].contiguous(), avg, towers)
        gr.lo, gr.hi = lo, hi
        ranks.append(gr)
    return whole, ranks, (table.data_ptr(), shift), table, bufs, src, dst


def check_ranks(emu, whole, ranks, peer, f0, fc):
    rc, gs_all, gb_all = whole.slots(emu.pna_aggregate_bwd_slots, f0, fc)
    assert rc == 0, emu.emu_last_error()
    out = []
    for gr in ranks:
        rc, gs, gb = gr.slots(emu.pna_aggregate_bwd_peer_slots, f0, fc, peer)
        assert rc == 0, emu.emu_last_error()
        s0, s1 = int(whole.rowptr[gr.lo]), int(whole.rowptr[gr.hi])
        assert torch.equal(gs[: gr.E], gs_all[s0:s1])                                    # every slot, bit for bit
        if whole.bias is not None:
            assert torch.equal(gb[:, f0:f0 + fc], gb_all[gr.lo:gr.hi, f0:f0 + fc])
        out.append(gs)
    return gs_all, out


CASES = [   # f, world, dtype, bias, towers, pad
    (12, 3, torch.float32, True, 1, 0), (8, 2, torch.float32, False, 1, 4), (75, 3, torch.float32, True, 1, 0),
    (75, 4, torch.float32, False, 3, 0), (160, 2, torch.float32, True, 2, 0), (16, 3, torch.bfloat16, True, 1, 0),
    (75, 2, torch.bfloat16, True, 1, 0), (40, 8, torch.bfloat16, False, 1, 8),
]


@pytest.mark.parametrize("f,world,dtype,with_bias,towers,pad", CASES)
def test_peer_slots_are_the_unpartitioned_per_slot_gradients(emu, f, world, dtype, with_bias, towers, pad):
    whole, ranks, peer, table, bufs, _, _ = setup(f, world, dtype, with_bias, towers, pad=pad)
    assert whole.hub_info.size(0) >= 1 and sum(gr.hub_info.size(0) for gr in ranks) >= 1    # a split row on some rank
    gs_all, _ = check_ranks(emu, whole, ranks, peer, 0, f)
    assert torch.isfinite(gs_all).all()


@pytest.mark.parametrize("f,world,dtype", [(40, 3, torch.float32), (75, 2, torch.float32), (48, 3, torch.bfloat16)])
def test_every_feature_slab_of_the_peer_slots(emu, f, world, dtype):
    whole, ranks, peer, *_ = setup(f, world, dtype, True, seed=4)
    al = 4 if dtype == torch.float32 else 8
    for width in (al, 2 * al, 3 * al):
        for f0 in range(0, f, width):
            check_ranks(emu, whole, ranks, peer, f0, min(width, f - f0))


def test_split_row_with_more_than_512_chunks(emu):
    """One destination with 4200 in-edges (526 chunks of 8) on the middle rank of three, fp32 and a row_bias."""
    whole, ranks, peer, *_ = setup(4, 3, torch.float32, True, n=60, e=300, big=4200, seed=2)
    assert int(whole.hub_info[:, 2].max()) > 512
    check_ranks(emu, whole, ranks, peer, 0, 4)


@pytest.mark.parametrize("f,world,dtype", [(12, 3, torch.float32), (75, 2, torch.float32), (16, 4, torch.bfloat16)])
def test_owners_pull_the_slots_in_whole_graph_slot_order(emu, emu_peer, f, world, dtype):
    """The gradient return: every owner adds the slots that gather its rows (its own included) with pna_halo_grad_pull on
    peer_grad_return_plans, starting from zero -- the sequential fp32 sum over the whole graph's slots in ascending order."""
    whole, ranks, peer, table, bufs, src, dst = setup(f, world, dtype, True, seed=7)
    gs_all, gss = check_ranks(emu, whole, ranks, peer, 0, f)
    plans = pd.peer_grad_return_plans([gr.col for gr in ranks], peer[1])
    e_max = max(gr.E for gr in ranks)
    staged = [torch.zeros(e_max, f) for _ in ranks]                    # the ranks' per-slot buffers, one pitch
    for s, gs in zip(staged, gss):
        s[: gs.size(0)] = gs[: s.size(0)]
    stable = torch.tensor([s.data_ptr() for s in staged], dtype=torch.int64)
    want = np.zeros((whole.n, f), dtype=np.float32)
    col, g = whole.col.numpy(), gs_all.numpy()
    for s in range(whole.E):
        want[col[s]] = want[col[s]] + g[s]
    for r, (gr, gp) in enumerate(zip(ranks, plans)):
        out = torch.zeros(gr.n, f)
        if gp.n_rows:
            rc = emu_peer.pna_halo_grad_pull(stable.data_ptr(), f, gp.rows.data_ptr(), gp.rowptr.data_ptr(), gp.enc.data_ptr(),
                                             gp.shift, gp.n_rows, out.data_ptr(), f, f, None)
            assert rc == 0, emu_peer.emu_last_error()
        assert torch.equal(out, torch.from_numpy(want[gr.lo:gr.hi])), r


def test_peer_slots_refusals(emu):
    whole, ranks, peer, *_ = setup(12, 2, torch.float32, True, seed=3)
    gr = ranks[0]
    fn = emu.pna_aggregate_bwd_peer_slots
    gs = torch.zeros(max(gr.E, 1), 12)

    def call(d, f0=0, fc=12, gs_=gs, ld=12):
        return fn(C.byref(d), gr.w.data_ptr(), gr.w.stride(0), f0, fc, None if gs_ is None else gs_.data_ptr(), ld, None, 0, None)
    assert call(gr.desc(None)) == PNA_ERR_BAD_ARG                        # no peer table
    d = gr.desc(peer)
    d.peer_shift = 0
    assert call(d) == PNA_ERR_BAD_ARG                                    # shift out of range
    d = gr.desc(peer)
    d.row_ids, d.n_row_ids = gr.col.data_ptr(), 1
    assert call(d) == PNA_ERR_UNSUPPORTED                                # row subsets
    d = gr.desc(peer)
    d.col = None
    assert call(d) == PNA_ERR_UNSUPPORTED                                # messages in CSR order: no owner to read from
    for aggr in ("moment3", "softmax", "softmin", "normalised_mean"):
        d = gr.desc(peer)
        d.n_aggr, d.aggr_codes = _lib.pack_codes(["mean", aggr], _lib.ALL_AGGR_CODES, "aggregator")
        assert call(d) == PNA_ERR_UNSUPPORTED, aggr
    for f0, fc in [(2, 4), (0, 0), (0, 13), (8, 8)]:                     # the slab rules of pna_aggregate_bwd_slots
        assert call(gr.desc(peer), f0, fc) == PNA_ERR_BAD_ARG, (f0, fc)
    assert call(gr.desc(peer), ld=8) == PNA_ERR_BAD_ARG                  # ld_grad_slots < f_count
    assert call(gr.desc(peer), gs_=None) == PNA_ERR_BAD_ARG              # no grad_slots
    assert torch.equal(gs, torch.zeros_like(gs))                         # nothing was written
    # the per-slot and atomic entry points keep refusing peer descriptors
    d = gr.desc(peer)
    assert emu.pna_aggregate_bwd_slots(C.byref(d), gr.w.data_ptr(), gr.w.stride(0), 0, 12, gs.data_ptr(), 12, None, 0, None) \
        == PNA_ERR_UNSUPPORTED
