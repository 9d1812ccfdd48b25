"""The add-on aggregators (moment3..5, softmax, softmin, normalised_mean) on the GPU against the exact fp32 restatement
(addon_paths_ref.py), with the device's own powf / expf bits injected from the probe oracle/devmath (built by build()).

Each case names the kernel instances it reaches (addon_paths_ref.addon_launches) and asserts a probe that shows the path
ran: split rows and their chunk counts, gridDim.y, the rows selected, the data edge it is about.  Outputs start as NaN.
Every element the kernels write must match bit for bit; bf16 outputs must be one round-to-nearest-even of the restated fp32
value; where the restatement gives NaN the kernel must give NaN.  Sums that atomics form (the atomic backward through col)
must lie within the order-free bound.  The scaler factors are the library's own (pna_row_scales).
"""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import addon_paths_ref as R
import backward_paths_ref as B
from test_gpu_backward_paths import _det, avg_of, host_of, rand, scales_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEVMATH = os.path.join(ROOT, "oracle", "_build", "libdevmath_sm90.so")
F32 = np.float32
S5 = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]
MIX6 = ["moment4", "softmin", "mean", "normalised_mean", "moment3", "softmax"]
SPLIT, CHUNK = 16, 4


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def P():
    import pna_b200
    return pna_b200


@pytest.fixture(scope="module")
def DM():
    if not os.path.exists(DEVMATH):
        pytest.fail(f"{DEVMATH} is missing: run __graft_entry__.build(), which builds the device-math probe")
    L = C.CDLL(DEVMATH)
    L.devmath_powf.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]
    L.devmath_expf.argtypes = [C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p]

    def run(fn, *arrays):
        ts = [torch.from_numpy(np.array(a, F32)).to(dev()) for a in arrays]
        out = torch.empty_like(ts[0])
        assert fn(*[t.data_ptr() for t in ts], out.data_ptr(), out.numel(), torch.cuda.current_stream().cuda_stream) == 0
        return out.cpu().numpy()
    return R.DevMath(lambda x, y: run(L.devmath_powf, x, y), lambda x: run(L.devmath_expf, x), "device")


def assert_same(got, want, what=""):
    g, w = np.ascontiguousarray(got, F32), np.ascontiguousarray(want, F32)
    gn, wn = np.isnan(g), np.isnan(w)
    assert (gn == wn).all(), f"{what}: NaN positions differ at {np.argwhere(gn != wn)[:4].tolist()}"
    bad = g.view(np.uint32)[~gn] != w.view(np.uint32)[~wn]
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ, first {np.argwhere(~gn)[bad][:4].tolist()}"


def as_dtype(a, dtype):
    return a if dtype == torch.float32 else torch.from_numpy(np.ascontiguousarray(a, F32)).to(torch.bfloat16).float().numpy()


def np32(t):
    return None if t is None else t.float().cpu().numpy()


# ---- graph: light rows of degree 0, 1, 2, split-1; split rows of degree split, k*chunk, k*chunk+1, and > 512 chunks -----
_G = {}


def graph(P):
    if "g" not in _G:
        rng = np.random.default_rng(7)
        n = 900
        k = SPLIT // CHUNK + 1
        fixed = {0: SPLIT - 1, 1: SPLIT, 2: k * CHUNK, 3: k * CHUNK + 1, 4: 1, 5: 2, 6: 6, 7: CHUNK * 520 + 3, 8: 5, 9: 40}
        dst = np.concatenate([rng.integers(20, n - 30, 2500)] + [np.full(d, r) for r, d in fixed.items()])
        src = rng.integers(0, n, dst.size)
        src[dst == 8] = 11          # rows 8 and 9 gather one source: identical messages
        src[dst == 9] = 11
        p = rng.permutation(dst.size)
        csr = P.build_csr(torch.from_numpy(src[p]).to(dev()), torch.from_numpy(dst[p]).to(dev()), n, SPLIT, CHUNK)
        _G["g"] = (csr, host_of(csr))
    return _G["g"]


def ref_graph(csr, host, col=True, dcol=None):
    return R.Graph(host[0], host[1] if col else None, host[2], csr.chunk_edges, csr.split_threshold, dcol=dcol)


def addon_cols(aggrs, F, towers, has_self, S):
    Ft, Wt, base = R.layout(F, towers, has_self, len(aggrs), S)
    cols = [base + (s * len(aggrs) + a) * Ft for a, nm in enumerate(aggrs) if R.code_of(nm) is not None for s in range(S)]
    return np.sort(np.concatenate(cols))


def probe_graph(csr, host):
    deg = np.diff(host[0])
    info = host[2]
    assert csr.n_hubs > 0 and int(info[:, 2].max()) > 512                      # split rows, one of more than 512 chunks
    assert {0, 4, 5} & set(info[:, 0].tolist()) == set() and {1, 2, 3, 7} <= set(info[:, 0].tolist())
    assert (deg == 0).any() and deg[0] == SPLIT - 1 and deg[2] % CHUNK == 0 and deg[3] % CHUNK == 1
    items = host[3]
    for h, (_, first, nch, _) in enumerate(info):                              # each split row's chunks are contiguous
        assert (items[first:first + nch, 0] == h).all() and (items[first:first + nch, 1] == np.arange(nch)).all()


# ---- 1. forward: widths, towers, self block, pitches, scalers ------------------------------------------------------------------
FWD = [
    # F, towers, self, dtype, layout, options        instances (gridDim.y)
    (1, 1, False, torch.float32, "contig", {}),             # k_mom_rows<float> + k_mom_chunk_*<float,4> + k_wsum_*: gy = 1, 1 active lane
    (31, 1, True, torch.float32, "pitch+2", {"sdeg": True}),  # partial warp, odd gathered pitch, scaler_degree
    (32, 2, False, torch.float32, "contig", {"zero": True}),  # full warp, zero_isolated
    (33, 3, True, torch.float32, "offset1", {}),              # gy = 2 (1 live lane in the second block), 3 towers + self
    (72, 3, True, torch.bfloat16, "pitch+2", {"sdeg": True}),  # bf16, gy = 3
    (160, 2, False, torch.float32, "contig", {}),             # gy = 5
]


def forward_case(P, DM, F, towers, has_self, dtype, layout, opt, aggrs=MIX6, ints=None, x=None, skip=None, bias=True):
    csr, host = graph(P)
    n = csr.n_nodes
    x = rand((n, F), dtype, F, layout, ints) if x is None else x
    b = rand((n, F), dtype, F + 1, ints=ints) if bias else None
    sf = rand((n, F), dtype, F + 2) if has_self else None
    avg = avg_of(csr)
    sdeg = None
    if opt.get("sdeg"):
        g = torch.Generator().manual_seed(F)
        sdeg = torch.randint(0, 30, (n,), generator=g, dtype=torch.int32)
        sdeg[::5] = 0
        sdeg = sdeg.to(dev())
    S = len(S5)
    width = towers * R.layout(F, towers, has_self, len(aggrs), S)[1]
    buf = torch.full((n, width + 3), float("nan"), dtype=dtype, device=dev())
    out = buf[:, :width]                                        # ld_out = width + 3: odd pitch
    P.aggregate.aggregate_forward(x, csr, aggrs, S5, avg, towers=towers, row_bias=b, self_feat=sf, zero_isolated=bool(opt.get("zero")),
                                  out=out, scaler_degree=sdeg, skip_light=skip == "light", skip_hubs=skip == "hubs")
    scales = scales_of(P, csr, S5, avg, sdeg)
    flags = (R.FLAG_ZERO_ISOLATED if opt.get("zero") else 0) | (R.FLAG_SKIP_LIGHT if skip == "light" else 0) | \
        (R.FLAG_SKIP_HUBS if skip == "hubs" else 0)
    want = R.forward(ref_graph(csr, host), np32(x), np32(b), aggrs, scales, DM, towers=towers, has_self=has_self, flags=flags)
    return out.float().cpu().numpy(), as_dtype(want, dtype), addon_cols(aggrs, F, towers, has_self, S)


@pytest.mark.parametrize("F,towers,has_self,dtype,layout,opt", FWD)
def test_forward_bit_for_bit(P, DM, F, towers, has_self, dtype, layout, opt):
    csr, host = graph(P)
    probe_graph(csr, host)
    L = R.addon_launches(MIX6, F, csr.n_nodes, csr.n_hubs, csr.n_chunks)
    assert dict(L)["k_mom_rows"][1] == -(-F // 32) and "k_wsum_hub_final[normalised_mean]" in dict(L)
    got, want, cols = forward_case(P, DM, F, towers, has_self, dtype, layout, opt)
    assert_same(got[:, cols], want[:, cols], "add-on columns")
    Ft, _, base = R.layout(F, towers, has_self, len(MIX6), len(S5))
    m3 = want[:, base + 4 * Ft]                                # moment3, identity scaler: both signs occur
    assert (m3 < 0).any() and (m3 > 0).any()


@pytest.mark.parametrize("skip", ["light", "hubs"])
def test_forward_row_selection(P, DM, skip):
    # SKIP_LIGHT: only the split-row chains (k_mom_chunk_* / k_wsum_chunk_*); SKIP_HUBS: only k_mom_rows / k_wsum_rows
    got, want, cols = forward_case(P, DM, 40, 1, False, torch.float32, "contig", {}, skip=skip)
    hub = ref_graph(*graph(P)).hub
    sel = hub if skip == "light" else ~hub
    assert_same(got[:, cols], want[:, cols], f"skip {skip}")
    assert np.isnan(got[~sel][:, cols]).all() and not np.isnan(got[sel][:, cols]).any()


@pytest.mark.parametrize("aggrs", [
    ["softmax", "moment5", "softmax", "max", "moment5", "sum"],                  # repeated add-ons: G sums over positions
    ["normalised_mean", "moment3", "softmin", "softmax"],                         # list order is not launch order
    ["normalised_mean", "softmax", "softmin", "moment3", "moment4", "moment5"],   # add-ons only, PNA_MAX_AGGR positions
])
def test_lists_forward_and_backward(P, DM, aggrs):
    got, want, cols = forward_case(P, DM, 24, 1, False, torch.float32, "contig", {}, aggrs=aggrs)
    assert_same(got[:, cols], want[:, cols], "forward")
    c = BwdCall(P, DM, 24, torch.float32, aggrs)
    c.check_slots()
    c.check_stores()
    c.check_python_atomic()


# ---- 2. backward ------------------------------------------------------------------------------------------------------------
class BwdCall:
    """One direct call into the backward ABI with the add-on codes, and the restatement of the same call."""

    def __init__(self, P, DM, F, dtype, aggrs, *, towers=1, has_self=False, layout="contig", go_extra=0, sdeg=False, ints=None,
                 x=None, bias=True):
        from pna_b200 import _lib
        self.P, self.L, self.lib = P, _lib.lib(), _lib
        self.csr, self.host = graph(P)
        n = self.csr.n_nodes
        self.F, self.dtype, self.aggrs, self.towers, self.has_self = F, dtype, aggrs, towers, has_self
        self.x = rand((n, F), dtype, 100 + F, layout, ints) if x is None else x.to(dtype)
        self.b = rand((n, F), dtype, 101 + F, ints=ints) if bias else None
        width = towers * R.layout(F, towers, has_self, len(aggrs), len(S5))[1]
        self.go = rand((n, width), dtype, 102 + F, ("wide", go_extra) if go_extra else "contig", ints)
        self.avg = avg_of(self.csr)
        self.sdeg = None
        if sdeg:
            g = torch.Generator().manual_seed(F)
            self.sdeg = torch.randint(0, 30, (n,), generator=g, dtype=torch.int32).to(dev())
        self.scales = scales_of(P, self.csr, S5, self.avg, self.sdeg)
        self.g = ref_graph(self.csr, self.host)
        self.gs, self.gb, self.terms = R.backward(self.g, np32(self.x), np32(self.b), np32(self.go), aggrs, self.scales, DM,
                                                  towers=towers, has_self=has_self)

    def desc(self, gathered, col, dcol=None):
        lib, csr = self.lib, self.csr
        na, ac = lib.pack_codes(self.aggrs, lib.ALL_AGGR_CODES, "aggregator")
        ns, sc = lib.pack_codes(S5, lib.SCALER_CODES, "scaler")
        self.scratch = torch.full(((csr.n_chunks + csr.n_hubs) * 6, self.F), float("nan"), device=dev())
        d = lib.AggStruct(
            gathered=gathered.data_ptr(), ld_gathered=gathered.stride(0), rowptr=csr.rowptr.data_ptr(), col=col,
            row_bias=None if self.b is None else self.b.data_ptr(), ld_row_bias=0 if self.b is None else self.b.stride(0),
            self_feat=1 if self.has_self else None, n_rows=csr.n_nodes, n_feat=self.F, n_towers=self.towers,
            dtype=lib.PNA_F32 if self.dtype == torch.float32 else lib.PNA_BF16, n_aggr=na, aggr_codes=ac, n_scalers=ns,
            scaler_codes=sc, avg_log=float(self.avg["log"]), avg_lin=float(self.avg["lin"]), split_threshold=csr.split_threshold,
            chunk_edges=csr.chunk_edges, hub_info=csr.hub_info.data_ptr(), chunk_items=csr.chunk_items.data_ptr(),
            n_hubs=csr.n_hubs, n_chunks=csr.n_chunks, hub_partials=self.scratch.data_ptr())
        if self.sdeg is not None:
            d.scaler_degree = self.sdeg.data_ptr()
        if dcol is not None:
            d.degree_col = dcol.data_ptr()
        return d

    def stream(self):
        return torch.cuda.current_stream().cuda_stream

    def check_slots(self, f0=0, fc=None, ld_extra=0):
        """pna_aggregate_bwd_slots over [f0, f0 + fc): grad_slots and grad_row_bias bit for bit, other columns untouched"""
        fc = self.F - f0 if fc is None else fc
        E, n = self.csr.n_edges, self.csr.n_nodes
        gs = torch.full((E, fc + ld_extra), float("nan"), device=dev())
        gb = torch.full((n, self.F), float("nan"), device=dev())
        d = self.desc(self.x, self.csr.col.data_ptr())
        self.lib.check(self.L.pna_aggregate_bwd_slots(C.byref(d), self.go.data_ptr(), self.go.stride(0), f0, fc, gs.data_ptr(),
                                                      fc + ld_extra, None if self.b is None else gb.data_ptr(), self.F, self.stream()))
        assert_same(gs[:, :fc].cpu().numpy(), self.gs[:, f0:f0 + fc], f"grad_slots [{f0}, +{fc})")
        if self.b is not None:
            gbn = gb.cpu().numpy()
            assert_same(gbn[:, f0:f0 + fc], self.gb[:, f0:f0 + fc], "grad_row_bias")
            assert np.isnan(np.delete(gbn, np.s_[f0:f0 + fc], axis=1)).all()
        return R.addon_launches(self.aggrs, fc, self.csr.n_nodes, self.csr.n_hubs, self.csr.n_chunks, backward=True)

    def check_stores(self):
        """pna_aggregate_bwd with col == NULL over the messages in CSR order, normalised_mean weighted through degree_col (the
        pretrans_layers > 1 layout): plain stores and adds, bit for bit"""
        xm = self.x[self.csr.col.long()].contiguous()
        dcol = self.csr.col.clone()
        E, n = self.csr.n_edges, self.csr.n_nodes
        gg = torch.full((E, self.F), float("nan"), device=dev())
        gb = torch.full((n, self.F), float("nan"), device=dev())
        d = self.desc(xm, None, dcol)
        self.lib.check(self.L.pna_aggregate_bwd(C.byref(d), self.go.data_ptr(), self.go.stride(0), gg.data_ptr(), self.F,
                                                None if self.b is None else gb.data_ptr(), self.F, self.stream()))
        assert_same(gg.cpu().numpy(), self.gs, "grad_gathered (col == NULL)")
        if self.b is not None:
            light = ~self.g.hub
            gbn = gb.cpu().numpy()
            assert_same(gbn[light], self.gb[light], "grad_row_bias, light rows")
            if all(R.code_of(a) is not None for a in self.aggrs):     # no core term: its atomic chunk shares are all 0
                assert_same(gbn, self.gb, "grad_row_bias")

    def check_atomic_col(self):
        """pna_aggregate_bwd through col: every term of every family lands by atomics, within the order-free bound"""
        n = self.csr.n_nodes
        gg = torch.zeros((n, self.F), device=dev())
        d = self.desc(self.x, self.csr.col.data_ptr())
        self.lib.check(self.L.pna_aggregate_bwd(C.byref(d), self.go.data_ptr(), self.go.stride(0), gg.data_ptr(), self.F, None, 0,
                                                self.stream()))
        rows = np.concatenate([self.host[1]] * len(self.terms))
        s, bound = B.order_free_sum(n, rows, np.concatenate([t for _, t in self.terms]))
        assert B.within_order_free(gg.cpu().numpy(), s, bound).all()

    def check_python_atomic(self):
        """aggregate_backward allocates grad_row_bias with torch.empty: every element must be written (the core kernels
        store it even when every core code is SKIP), over a block that held NaN"""
        junk = torch.full((self.csr.n_nodes, self.F), float("nan"), device=dev())
        del junk
        gg, gb = self.P.aggregate.aggregate_backward(self.go, self.x, self.csr, self.aggrs, S5, self.avg, row_bias=self.b,
                                                     need_bias_grad=True)
        gbn = gb.cpu().numpy()
        light = ~self.g.hub
        assert_same(gbn[light], self.gb[light], "grad_row_bias (Python, atomic), light rows")
        assert not np.isnan(gbn).any()
        if all(R.code_of(a) is not None for a in self.aggrs):
            assert_same(gbn, self.gb, "grad_row_bias (Python, atomic)")


BWD = [
    # F, towers, self, dtype, layout, go_extra, sdeg      instances (per-slot: k_mom_bwd_rows<T,true>, k_mom_bwd_chunk_grad<T,true>,
    #                                                      k_wsum_bwd_*<T,true>, k_mom_bwd_hub_bias<6>; gridDim.y of the slab)
    (1, 1, False, torch.float32, "contig", 0, False),
    (31, 1, True, torch.float32, "pitch+2", 3, True),
    (33, 3, True, torch.float32, "offset1", 0, False),
    (72, 3, True, torch.bfloat16, "pitch+2", 1, True),
    (160, 2, False, torch.float32, "contig", 0, False),
    (64, 2, True, torch.bfloat16, "contig", 0, False),
]


@pytest.mark.parametrize("F,towers,has_self,dtype,layout,go_extra,sdeg", BWD)
def test_backward_bit_for_bit(P, DM, F, towers, has_self, dtype, layout, go_extra, sdeg):
    c = BwdCall(P, DM, F, dtype, MIX6, towers=towers, has_self=has_self, layout=layout, go_extra=go_extra, sdeg=sdeg)
    L = c.check_slots()
    assert dict(L)["k_mom_bwd_rows"][1] == -(-F // 32) and "k_mom_bwd_hub_bias<6>" in dict(L)
    al = 4 if dtype == torch.float32 else 8
    if F > 2 * al:                                       # slabs: f0 > 0 (gridDim.y of the slab), and the ragged last one
        L = c.check_slots(al, 2 * al if F < 64 else 40, ld_extra=1)
        assert dict(L)["k_mom_bwd_rows"][1] == (1 if F < 64 else 2)
        c.check_slots((F - 1) // al * al)
    c.check_stores()
    c.check_atomic_col()


@pytest.mark.parametrize("F,dtype", [(64, torch.float32), (72, torch.bfloat16)])
def test_deterministic_path_through_python(P, DM, F, dtype):
    """under torch.use_deterministic_algorithms: per-slot rows, then the forward 'sum' over the slot-transposed CSR"""
    c = BwdCall(P, DM, F, dtype, MIX6)
    csr = c.csr
    tcsr = csr.slot_transposed(csr.n_nodes)
    gg, gb = _det(lambda: P.aggregate.aggregate_backward(c.go, c.x, csr, MIX6, S5, c.avg, row_bias=c.b, need_bias_grad=True))
    w = P.aggregate.deterministic_slab_width(csr.n_edges, F, 16 // c.x.element_size())
    want = np.empty((csr.n_nodes, F), F32)
    for f0 in range(0, F, w):
        fc = min(w, F - f0)
        want[:, f0:f0 + fc], _ = B.transposed_sums(np.ascontiguousarray(c.gs[:, f0:f0 + fc]), host_of(tcsr), tcsr.chunk_edges, fc,
                                                   fc % 4 == 0 and F % 4 == 0)
    assert_same(gg.cpu().numpy(), want, "deterministic grad_gathered")
    assert_same(gb.cpu().numpy(), c.gb, "deterministic grad_row_bias")


# ---- 3. data edges ------------------------------------------------------------------------------------------------------------
def _ulp_ints(n, F, lo, hi, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(lo, hi, (n, F), generator=g).double() * 2.0 ** -149).float().to(dev())


def test_identical_messages_pass_zero_through(P, DM):
    """rows 8 and 9 (light, split) gather one source: integer data makes delta = 0 exactly, M_k = 0, r_k = 0 and the slope 0"""
    csr, host = graph(P)
    got, want, cols = forward_case(P, DM, 32, 1, False, torch.float32, "contig", {}, ints=3)
    assert_same(got[:, cols], want[:, cols], "forward")
    Ft, _, base = R.layout(32, 1, False, len(MIX6), len(S5))
    mom_cols = np.concatenate([base + (s * len(MIX6) + a) * Ft for a in (0, 4) for s in range(len(S5))])   # moment4, moment3
    assert (want[[8, 9]][:, mom_cols] == 0).all() and 9 in host[2][:, 0] and 8 not in host[2][:, 0]
    c = BwdCall(P, DM, 32, torch.float32, MIX6, ints=3)
    c.check_slots()
    c.check_stores()


def test_subnormal_row_sums(P, DM):
    """messages that are small multiples of 2^-149: every mean is a subnormal quotient, some of them exact ties, where a
    reciprocal-and-correction division (SharedDivisor) can miss the correctly rounded result"""
    csr, host = graph(P)
    x = _ulp_ints(csr.n_nodes, 32, -40, 41, 5)
    got, want, cols = forward_case(P, DM, 32, 1, False, torch.float32, "contig", {}, x=x, aggrs=["moment3", "moment4", "softmax"],
                                   bias=False)
    assert_same(got[:, cols], want[:, cols], "forward")
    # the probe: the restated sums include quotients where fl(q + fl(e r)) with q = fl(x fl(1/d)) differs from x / d
    g = ref_graph(csr, host)
    m = g.messages(np32(x), None)
    S, _ = g.row_sums(m)
    d = np.maximum(g.deg, 1).astype(F32)[:, None]
    r = F32(1) / d
    q = S * r
    markstein = B.fma32(B.fma32(-q, np.broadcast_to(d, q.shape), S), np.broadcast_to(r, q.shape), q)
    assert (markstein != S / d).any()
    c = BwdCall(P, DM, 32, torch.float32, ["moment3", "moment5", "mean"], x=x, bias=False)
    c.check_slots()


def test_fifth_powers_that_overflow(P, DM):
    """|delta| ~ 1e8: delta^5 overflows, M_5 is +-inf or NaN (inf - inf); the restatement defines what the kernels give"""
    csr, host = graph(P)
    x = (rand((csr.n_nodes, 32), torch.float32, 9) * 1e8).contiguous()
    got, want, cols = forward_case(P, DM, 32, 1, False, torch.float32, "contig", {}, x=x, aggrs=["moment5", "moment3", "softmin"])
    r5 = want[:, cols][:, :32]
    assert np.isinf(r5).any() and np.isnan(r5).any()         # the probe: both kinds of row occur
    assert_same(got[:, cols], want[:, cols], "forward")
    c = BwdCall(P, DM, 32, torch.float32, ["moment5", "moment3", "softmin"], x=x, bias=False)
    c.check_slots()
    c.check_stores()


def test_softmax_rows_where_most_weights_underflow(P, DM):
    """messages spanning ~200: most expf(n - M) are 0"""
    csr, host = graph(P)
    x = (rand((csr.n_nodes, 33), torch.float32, 12) * 60).contiguous()
    c = BwdCall(P, DM, 33, torch.float32, ["softmax", "softmin", "moment3"], x=x)
    m = c.g.messages(np32(c.x), np32(c.b))
    e = DM.expf(m - c.g.row_max(m)[c.g.row])
    assert (e == 0).mean() > 0.3
    got, want, cols = forward_case(P, DM, 33, 1, False, torch.float32, "contig", {}, x=x, aggrs=["softmax", "softmin", "moment3"])
    assert_same(got[:, cols], want[:, cols], "forward")
    c.check_slots()
    c.check_stores()


# ---- 4. the probe itself -------------------------------------------------------------------------------------------------------
def test_devmath_probe_within_the_documented_ulp_bounds(DM):
    """a sanity check of the probe, not the bar: powf within 4 ulp, expf within 2 ulp (CUDA Math API) of float64"""
    x = np.geomspace(1e-5, 1e30, 4001).astype(F32)
    for y in list(R.INV_K.values()) + list(R.SLOPE_E.values()):
        got = DM.powf(x, np.full_like(x, y))
        want = np.power(x.astype(np.float64), float(y))
        ulp = np.spacing(want.astype(F32)).astype(np.float64)
        assert (np.abs(got - want) <= 4 * ulp).all(), y
    x = np.linspace(-100, 88, 20001).astype(F32)
    got, want = DM.expf(x), np.exp(x.astype(np.float64))
    assert (np.abs(got - want) <= 2 * np.spacing(want.astype(F32)).astype(np.float64)).all()
