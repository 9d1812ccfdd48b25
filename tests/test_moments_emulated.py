"""The moment kernels (csrc/pna_aggregate_moments.cuh) executed on the HOST, thread by thread (tests/emu), through the real C
entry points pna_aggregate_fwd / pna_aggregate_bwd / pna_aggregate_bwd_slots.  The existing aggregation kernels use shared
memory and shuffles and are not emulated: here they are stubbed out, so every non-moment column and gradient is left as it
was -- which also checks that the moment kernels write nothing else.  Light rows must equal the C oracle bit for bit; split
rows (chunk-parallel, fixed merge order) must be within the bar of tests/moment_bars.py and identical across runs."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

import moment_oracle as MO
from pna_b200 import _lib
import moment_bars as MB

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

HERE = os.path.dirname(os.path.abspath(__file__))
SPLIT, CHUNK = 16, 8
SCALERS = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]
PNA_ERR_UNSUPPORTED = -2

_STUBS = """
namespace pna {
// the existing forward kernels (shared memory, shuffles) are not emulated: they write nothing here
template <typename T, int VEC> int launch_typed(const KParams&, cudaStream_t) { return PNA_OK; }
static thread_local char g_err[512];
void set_error(const char* fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof(g_err), fmt, ap); va_end(ap); }
int cuda_fail(cudaError_t, const char* what) { set_error("%s", what); return PNA_ERR_CUDA; }
}
extern "C" int pna_query(int what) { return what == PNA_QUERY_MAX_FEATURES ? 16384 : 0; }
extern "C" const char* emu_last_error(void) { return pna::g_err; }
"""


def _build():
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    asan = os.environ.get("PNA_EMU_ASAN") == "1"
    srcs = [os.path.join(be.CSRC, n) for n in ("pna_aggregate.cu", "pna_aggregate_bwd.cu")]
    deps = srcs + [os.path.join(be.CSRC, n) for n in ("pna_aggregate.cuh", "pna_aggregate_moments.cuh", "common.cuh")] + [
        os.path.join(be.HERE, "cuda_host_shim.h"), os.path.join(be.ROOT, "include", "pna_b200.h"), __file__]
    os.makedirs(be.BUILD, exist_ok=True)
    lib = os.path.join(be.BUILD, f"libmoments_emu{'_asan' if asan else ''}.so")
    if os.path.exists(lib) and all(os.path.getmtime(lib) >= os.path.getmtime(d) for d in deps):
        return lib
    body = ""
    for s in srcs:
        t = be.strip_inline_ptx(be.rewrite_launches(open(s).read()))
        body += re.sub(r'#include "(pna_aggregate\.cuh|common\.cuh)"', lambda m: f'#include "{be.CSRC}/{m.group(1)}"', t) + "\n"
    tu = os.path.join(be.BUILD, "moments_emu.cpp")
    with open(tu, "w") as f:
        f.write(f'#include "{be.HERE}/cuda_host_shim.h"\n#include <stdarg.h>\n#include <stdio.h>\n')
        f.write(body)
        f.write(_STUBS)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = ["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-w", f"-I{cuda_inc}", tu, "-o", lib]
    if asan:
        cmd[1:1] = ["-g", "-fsanitize=address", "-fno-omit-frame-pointer"]
    subprocess.run(cmd, check=True)
    return lib


@pytest.fixture(scope="module")
def emu():
    try:
        L = C.CDLL(_build())
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    L.pna_aggregate_fwd.argtypes = [C.POINTER(_lib.AggStruct), C.c_void_p]
    L.pna_aggregate_bwd.argtypes = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64,
                                    C.c_void_p]
    L.pna_aggregate_bwd_slots.argtypes = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p,
                                          C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    L.pna_aggregate_bwd_coef.argtypes = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_int32,
                                         C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    return L


def graph(n, e, seed, big=0, huge=0):
    """Random multigraph with duplicates and self loops; the last 5 rows are isolated; rows 0-3 get exactly 1 in-edge;
    `big` slots go to row 5 (a split row) and `huge` to row 6."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(10, n - 5, (e,), generator=g)
    src[:6] = dst[:6]                                   # self loops
    src[6:10] = src[10]; dst[6:10] = dst[10]            # duplicates
    extra_s = [torch.randint(0, n, (4,), generator=g)]
    extra_d = [torch.arange(4)]                          # d = 1
    if big:
        extra_s.append(torch.randint(0, n, (big,), generator=g)); extra_d.append(torch.full((big,), 5))
    if huge:
        extra_s.append(torch.randint(0, n, (huge,), generator=g)); extra_d.append(torch.full((huge,), 6))
    return torch.cat([src] + extra_s), torch.cat([dst] + extra_d), g


class Case:
    def __init__(self, emu, n, e, F, seed, dtype=torch.float32, towers=1, bias=True, self_feat=False, big=70, huge=0,
                 aggrs=("mean", "moment3", "max", "moment4", "moment5"), scalers=("identity", "amplification"), sdeg=False):
        self.emu, self.n, self.F, self.towers, self.dtype = emu, n, F, towers, dtype
        self.src, self.dst, g = graph(n, e, seed, big, huge)
        self.x = (torch.randn(n, F, generator=g) * 2 + 0.5).to(dtype)
        self.bias = torch.randn(n, F, generator=g).to(dtype) if bias else None
        self.self_feat = torch.randn(n, F, generator=g).to(dtype) if self_feat else None
        self.aggrs, self.scalers = list(aggrs), list(scalers)
        order = torch.sort(self.dst, stable=True).indices
        self.col = self.src[order].to(torch.int32).contiguous()
        self.deg = torch.bincount(self.dst, minlength=n)
        self.rowptr = torch.zeros(n + 1, dtype=torch.int32)
        self.rowptr[1:] = torch.cumsum(self.deg, 0).to(torch.int32)
        hubs, chunks = [], []
        for r in (self.deg >= SPLIT).nonzero().flatten().tolist():
            nch = (int(self.deg[r]) + CHUNK - 1) // CHUNK
            hubs.append([r, len(chunks), nch, int(self.deg[r])])
            chunks += [[len(hubs) - 1, j] for j in range(nch)]
        self.hub_info = torch.tensor(hubs, dtype=torch.int32).reshape(-1, 4).contiguous()
        self.chunk_items = torch.tensor(chunks, dtype=torch.int32).reshape(-1, 2).contiguous()
        self.sdeg = ((self.deg + torch.arange(n) % 3).to(torch.int32).contiguous()) if sdeg else None
        self.avg = {"log": 1.7, "lin": 4.5}
        self.A, self.S = len(self.aggrs), len(self.scalers)
        self.Ft = F // towers
        self.W = towers * ((1 if self_feat else 0) + self.A * self.S) * self.Ft

    def desc(self, out=None, flags=0, scratch_rows=4):
        na, ac = _lib.pack_codes(self.aggrs, _lib.ALL_AGGR_CODES, "aggregator")
        ns, sc = _lib.pack_codes(self.scalers, _lib.SCALER_CODES, "scaler")
        nh, nc = self.hub_info.size(0), self.chunk_items.size(0)
        self.scratch = torch.full(((nc + (nh if scratch_rows == 6 else 0)) * scratch_rows, self.F), float("nan"))
        b, s = self.bias, self.self_feat
        d = _lib.AggStruct(
            gathered=self.x.data_ptr(), ld_gathered=self.F, rowptr=self.rowptr.data_ptr(), col=self.col.data_ptr(),
            row_bias=None if b is None else b.data_ptr(), ld_row_bias=0 if b is None else self.F,
            self_feat=None if s is None else s.data_ptr(), ld_self=0 if s is None else self.F,
            self_tower_stride=self.Ft if s is not None else 0,
            out=None if out is None else out.data_ptr(), ld_out=self.W,
            n_rows=self.n, n_feat=self.F, n_towers=self.towers, dtype=_lib.PNA_F32 if self.dtype == torch.float32 else _lib.PNA_BF16,
            n_aggr=na, aggr_codes=ac, n_scalers=ns, scaler_codes=sc, avg_log=self.avg["log"], avg_lin=self.avg["lin"],
            flags=flags, split_threshold=SPLIT, chunk_edges=CHUNK,
            hub_info=self.hub_info.data_ptr() if nh else None, chunk_items=self.chunk_items.data_ptr() if nh else None,
            n_hubs=nh, n_chunks=nc, hub_partials=self.scratch.data_ptr() if self.scratch.numel() else None)
        if self.sdeg is not None:
            d.scaler_degree = self.sdeg.data_ptr()
        return d

    def forward(self, flags=0, view_mask=None):
        out = torch.full((self.n, self.W), float("nan")).to(self.dtype)
        d = self.desc(out, flags)
        keep = []
        if view_mask is not None:       # a masked light view in row order: light_deg = -1 outside the mask
            ldeg = torch.where(view_mask & (self.deg < SPLIT), self.deg, torch.full_like(self.deg, -1)).to(torch.int32).contiguous()
            lrp = torch.zeros(self.n + 1, dtype=torch.int32)
            part = torch.tensor([0, self.n], dtype=torch.int32)
            keep = [ldeg, lrp, part, self.col]
            d.light_rowptr, d.light_deg, d.light_col, d.part, d.n_part = lrp.data_ptr(), ldeg.data_ptr(), self.col.data_ptr(), part.data_ptr(), 1
            d.n_view_rows = self.n
        rc = self.emu.pna_aggregate_fwd(C.byref(d), None)
        assert rc == 0, self.emu.emu_last_error()
        del keep
        return out

    def messages(self):
        """fp32 per-edge messages in edge order, exactly as the kernel forms them."""
        m = self.x.float()[self.src]
        return m + self.bias.float()[self.dst] if self.bias is not None else m

    def column(self, out, t, s, a):
        """[n, Ft] block of (tower t, scaler s, aggregator a)."""
        has_self = self.self_feat is not None
        base = t * (self.W // self.towers) + (self.Ft if has_self else 0) + (s * self.A + a) * self.Ft
        return out[:, base:base + self.Ft].float()


def same_bits(a, b):
    """Bitwise equality (the untouched columns hold NaN)."""
    it = torch.int32 if a.dtype == torch.float32 else torch.int16
    return torch.equal(a.view(it), b.view(it))


def expected(c: Case):
    """C oracle r_k per moment position, per tower ([n, F], unscaled)."""
    msg = c.messages()
    ei = torch.stack([torch.arange(msg.size(0)), c.dst])
    return {k: MO.moment(msg, ei, c.n, k) for k in (3, 4, 5)}


def check_forward(c: Case, out, rows):
    """Light rows in `rows`: bit-identical to the C oracle (identity column) and scaled columns; split rows: within the bar."""
    want = expected(c)
    msg = c.messages()
    light = rows & (c.deg < SPLIT)
    hub = rows & (c.deg >= SPLIT)
    for a, name in enumerate(c.aggrs):
        if not name.startswith("moment"):
            continue
        k = int(name[-1])
        r64, tol = MB.moment_bar(msg, c.dst, c.n, k)
        for t in range(c.towers):
            sl = slice(t * c.Ft, (t + 1) * c.Ft)
            ident = c.column(out, t, 0, a)
            w = want[k][:, sl]
            if c.dtype == torch.bfloat16:
                w = w.to(torch.bfloat16).float()
            assert torch.equal(ident[light], w[light]), (name, t)
            err = (ident[hub] - r64[:, sl][hub]).abs()
            lim = tol[:, sl][hub] + (r64[:, sl][hub].abs() * 2.0 ** -8 if c.dtype == torch.bfloat16 else 0)
            assert (err <= lim).all(), (name, t, float((err / lim).max()))
            for s in range(1, c.S):
                col = c.column(out, t, s, a)
                want_s = ident * scale_factor(c, c.scalers[s]).unsqueeze(1).float()
                rt = 1e-6 if c.dtype == torch.float32 else 2.0 ** -7
                torch.testing.assert_close(col[rows], want_s[rows], rtol=rt, atol=0)


def scale_factor(c, name):
    """Scaler factor per row (scalers.py:8-29) at the scalers' degree, float64."""
    d = (c.sdeg if c.sdeg is not None else c.deg).double()
    lg = torch.log(d + 1)
    one = torch.ones_like(d)
    return {"identity": one, "amplification": lg / c.avg["log"],
            "attenuation": torch.where(d > 0, c.avg["log"] / lg, one), "linear": d / c.avg["lin"],
            "inverse_linear": torch.where(d > 0, c.avg["lin"] / d, one)}[name]


@pytest.mark.parametrize("F,towers,dtype,bias,self_feat,sdeg", [
    (12, 1, torch.float32, True, False, False), (16, 2, torch.float32, True, True, False), (10, 1, torch.float32, False, False, True),
    (40, 4, torch.float32, True, True, True), (16, 1, torch.bfloat16, True, False, False), (24, 3, torch.bfloat16, True, True, True),
])
def test_forward_matches_the_c_oracle_and_the_bar(emu, F, towers, dtype, bias, self_feat, sdeg):
    c = Case(emu, 60, 400, F, seed=F + towers, dtype=dtype, towers=towers, bias=bias, self_feat=self_feat, sdeg=sdeg,
             scalers=SCALERS)
    assert c.hub_info.size(0) >= 1 and (c.deg == 0).sum() >= 5 and (c.deg == 1).sum() >= 4
    out = c.forward()
    rows = torch.ones(c.n, dtype=torch.bool)
    check_forward(c, out, rows)
    # isolated rows: every moment column is 0, for every scaler
    for a, name in enumerate(c.aggrs):
        for t in range(towers):
            for s in range(c.S):
                col = c.column(out, t, s, a)
                if name.startswith("moment"):
                    assert torch.equal(col[c.deg == 0], torch.zeros_like(col[c.deg == 0]))
                else:      # the stubbed main path wrote nothing: the moment kernels touch only their own columns
                    assert torch.isnan(col).all()
    if self_feat:
        blocks = out.float().view(c.n, towers, -1)[:, :, :c.Ft]
        assert torch.isnan(blocks).all()
    assert same_bits(c.forward(), out)                                     # same bits on every run


def test_split_row_with_more_than_512_chunks(emu):
    c = Case(emu, 40, 150, 4, seed=3, big=40, huge=CHUNK * 520 + 3, aggrs=("moment3", "moment4", "moment5"),
             scalers=("identity",))
    assert int(c.hub_info[:, 2].max()) > 512
    out = c.forward()
    check_forward(c, out, torch.ones(c.n, dtype=torch.bool))
    assert same_bits(c.forward(), out)


def test_row_selection_skip_light_skip_hubs_and_masked_view(emu):
    c = Case(emu, 60, 400, 12, seed=8)
    light, hub = c.deg < SPLIT, c.deg >= SPLIT
    moment_cols = torch.zeros(c.W, dtype=torch.bool)
    for a, name in enumerate(c.aggrs):
        if name.startswith("moment"):
            for s in range(c.S):
                moment_cols[(s * c.A + a) * c.Ft:(s * c.A + a + 1) * c.Ft] = True
    for flags, rows in ((_lib.FLAG_SKIP_LIGHT, hub), (_lib.FLAG_SKIP_HUBS, light)):
        out = c.forward(flags)
        check_forward(c, out, rows)
        assert torch.isnan(out[~rows]).all()
        assert torch.isfinite(out[rows][:, moment_cols]).all()
    mask = torch.arange(c.n) % 2 == 0
    out = c.forward(view_mask=mask)
    sel = (mask & light) | hub
    check_forward(c, out, sel)
    assert torch.isnan(out[~sel]).all()


# ---- backward ----------------------------------------------------------------------------------------------------------
def run_bwd(c: Case, go, slots, f0=0, fc=None):
    fc = c.F if fc is None else fc
    E = c.col.numel()
    d = c.desc(scratch_rows=6)
    gb = torch.full((c.n, c.F), 0.25) if c.bias is not None else None
    go = go.to(c.dtype).contiguous()
    if slots:
        gs = torch.full((E, fc), 0.5)          # what the (stubbed) per-slot kernel would have stored
        rc = c.emu.pna_aggregate_bwd_slots(C.byref(d), go.data_ptr(), c.W, f0, fc, gs.data_ptr(), fc,
                                           None if gb is None else gb.data_ptr(), c.F, None)
        assert rc == 0, c.emu.emu_last_error()
        return gs, gb
    gg = torch.full((E, c.F), 0.5)             # col == NULL: per-slot rows of the materialised messages
    xm = c.x[c.col.long()].contiguous()
    bm = c.bias
    d.gathered, d.col = xm.data_ptr(), None
    rc = c.emu.pna_aggregate_bwd(C.byref(d), go.data_ptr(), c.W, gg.data_ptr(), c.F, None if gb is None else gb.data_ptr(),
                                 c.F, None)
    assert rc == 0, c.emu.emu_last_error()
    del xm, bm
    return gg, gb


MOM3 = ("moment4", "moment3", "moment5")


@pytest.mark.parametrize("F,towers,dtype,bias,aggrs", [
    (12, 1, torch.float32, True, MOM3), (16, 2, torch.float32, False, MOM3), (40, 4, torch.float32, True, MOM3),
    (8, 1, torch.float32, True, ("moment3", "moment3")), (12, 1, torch.float32, True, ("moment5",)),
    (16, 1, torch.bfloat16, True, MOM3), (24, 3, torch.bfloat16, True, ("moment4",))])
def test_backward_atomic_and_slots_agree_and_match_float64(emu, F, towers, dtype, bias, aggrs):
    """Moments only: the existing kernels (run for real here) then store a zero gradient for every slot, so what the
    buffers hold afterwards is the moment term alone."""
    c = Case(emu, 60, 400, F, seed=20 + F, dtype=dtype, towers=towers, bias=bias, aggrs=aggrs, scalers=("identity", "attenuation"))
    go = torch.randn(c.n, c.W, generator=torch.Generator().manual_seed(F))
    gs, gb = run_bwd(c, go, slots=True)
    ga, gba = run_bwd(c, go, slots=False)
    assert torch.equal(gs, ga)                                 # the same value of every slot in both instances
    if bias:
        assert torch.equal(gb, gba)
    assert torch.equal(run_bwd(c, go, slots=True)[0], gs)       # and the same bits on every run
    # slab = column slice of the full-width run
    al = 4 if dtype == torch.float32 else 8
    if F > al:
        gs2, _ = run_bwd(c, go, slots=True, f0=al, fc=min(al, F - al))
        assert torch.equal(gs2, gs[:, al:al + gs2.size(1)])
    # against float64 autograd, per slot, and summed per source row / destination row
    msg = c.messages()
    order = torch.sort(c.dst, stable=True).indices
    go_f = go.to(dtype).float()
    for t in range(towers):
        sl = slice(t * c.Ft, (t + 1) * c.Ft)
        G = {}
        for a, name in enumerate(c.aggrs):
            if name.startswith("moment"):
                k = int(name[-1])
                sdeg = c.deg.float()
                lg = torch.log(sdeg + 1)
                att = torch.where(sdeg > 0, c.avg["log"] / lg, torch.ones_like(lg)).unsqueeze(1)
                G[k] = G.get(k, 0) + c.column(go_f, t, 0, a) + att * c.column(go_f, t, 1, a)
        g64, tol = MB.moment_grad_bar(msg[:, sl], c.dst, c.n, sorted(G), G)
        term = gs[:, sl]                                       # CSR slot order
        err = (term - g64[order].float()).abs()
        lim = tol[order].float()
        assert (err <= lim).all(), float((err / lim).nan_to_num(0).max())
        # in-order sums (per source row, and grad_row_bias per destination): the per-slot bars add up, plus one rounding
        # per fp32 add, bounded by E * u * sum |g|
        for idx, got in ((c.col.long(), None), (c.dst[order], gb[:, sl] if bias else None)):
            want = torch.zeros(c.n, c.Ft, dtype=torch.float64).index_add(0, idx, g64[order])
            if got is None:
                got = torch.zeros(c.n, c.Ft)
                for e in range(term.size(0)):                   # ascending slot order, fp32 adds
                    got[idx[e]] = got[idx[e]] + term[e]
            bound = torch.zeros_like(want).index_add(0, idx, tol[order]) + \
                torch.zeros_like(want).index_add(0, idx, g64[order].abs()) * term.size(0) * MB.U
            assert ((got.double() - want).abs() <= bound).all()


def test_coef_row_ids_and_peer_refuse_moments(emu):
    c = Case(emu, 30, 100, 8, seed=2, big=0)
    out = torch.zeros(c.n, c.W)
    d = c.desc(out)
    ids = torch.arange(3, dtype=torch.int32)
    d.row_ids, d.n_row_ids = ids.data_ptr(), 3
    assert emu.pna_aggregate_fwd(C.byref(d), None) == PNA_ERR_UNSUPPORTED
    d = c.desc(out)
    d.peer_gathered, d.peer_shift = 256, 8
    assert emu.pna_aggregate_fwd(C.byref(d), None) == PNA_ERR_UNSUPPORTED
    assert torch.equal(out, torch.zeros_like(out))
    d = c.desc(scratch_rows=6)
    go = torch.zeros(c.n, c.W)
    coef = torch.zeros(c.n, 2 * c.F)
    gg = torch.zeros(c.n, c.F)
    rc = emu.pna_aggregate_bwd_coef(C.byref(d), go.data_ptr(), c.W, coef.data_ptr(), 2 * c.F, c.F, gg.data_ptr(), c.F, None, 0, None)
    assert rc == PNA_ERR_UNSUPPORTED
    assert b"coefficient" in emu.emu_last_error()
    d.row_ids, d.n_row_ids = ids.data_ptr(), 3
    rc = emu.pna_aggregate_bwd(C.byref(d), go.data_ptr(), c.W, gg.data_ptr(), c.F, None, 0, None)
    assert rc == PNA_ERR_UNSUPPORTED
