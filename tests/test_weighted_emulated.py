"""The softmax / softmin / normalised_mean kernels (csrc/pna_aggregate_weighted.cuh) executed on the HOST, thread by thread
(tests/emu), through the real C entry points pna_aggregate_fwd / pna_aggregate_bwd / pna_aggregate_bwd_slots.  As in
tests/test_moments_emulated.py the existing forward kernels are stubbed out, so every other column is left as it was --
which also checks that these kernels write nothing else; the existing backward kernels run and store a zero gradient for
every slot (their list holds only PNA_AGGR_SKIP).  Light rows must equal the C oracle bit for
bit; split rows (chunk-parallel, fixed merge order) must be within the bar of tests/weighted_bars.py and identical across
runs."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest
import torch

import weighted_bars as WB
import weighted_oracle as WO
from pna_b200 import _lib
from test_moments_emulated import CHUNK, SCALERS, SPLIT, Case, _STUBS, same_bits, scale_factor

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

HERE = os.path.dirname(os.path.abspath(__file__))
PNA_ERR_UNSUPPORTED = -2
WEIGHTED = ("softmax", "softmin", "normalised_mean")


def _build():
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    asan = os.environ.get("PNA_EMU_ASAN") == "1"
    srcs = [os.path.join(be.CSRC, n) for n in ("pna_aggregate.cu", "pna_aggregate_bwd.cu")]
    deps = srcs + [os.path.join(be.CSRC, n) for n in ("pna_aggregate.cuh", "pna_aggregate_moments.cuh",
                                                      "pna_aggregate_weighted.cuh", "common.cuh")] + [
        os.path.join(be.HERE, "cuda_host_shim.h"), os.path.join(be.ROOT, "include", "pna_b200.h"), __file__]
    os.makedirs(be.BUILD, exist_ok=True)
    lib = os.path.join(be.BUILD, f"libweighted_emu{'_asan' if asan else ''}.so")
    if os.path.exists(lib) and all(os.path.getmtime(lib) >= os.path.getmtime(d) for d in deps):
        return lib
    body = ""
    for s in srcs:
        t = be.strip_inline_ptx(be.rewrite_launches(open(s).read()))
        body += re.sub(r'#include "(pna_aggregate\.cuh|common\.cuh)"', lambda m: f'#include "{be.CSRC}/{m.group(1)}"', t) + "\n"
    tu = os.path.join(be.BUILD, "weighted_emu.cpp")
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


MIX = ("mean", "softmax", "max", "normalised_mean", "softmin")


def check_forward(c: Case, out, rows):
    """Light rows in `rows`: bit-identical to the C oracle (identity column) and scaled columns; split rows: within the bar."""
    msg = c.messages()
    light = rows & (c.deg < SPLIT)
    hub = rows & (c.deg >= SPLIT)
    for a, name in enumerate(c.aggrs):
        if name not in WEIGHTED:
            continue
        want = WO.weighted(msg, c.dst, c.n, name, wsrc=c.src)
        y64, tol = WB.bar(name, msg, c.dst, c.n, wsrc=c.src)
        for t in range(c.towers):
            sl = slice(t * c.Ft, (t + 1) * c.Ft)
            ident = c.column(out, t, 0, a)
            w = want[:, sl]
            if c.dtype == torch.bfloat16:
                w = w.to(torch.bfloat16).float()
            assert torch.equal(ident[light], w[light]), (name, t)
            err = (ident[hub].double() - y64[:, sl][hub]).abs()
            lim = tol[:, sl][hub] + (y64[:, sl][hub].abs() * 2.0 ** -8 if c.dtype == torch.bfloat16 else 0)
            assert (err <= lim).all(), (name, t, float((err / lim).max()))
            for s in range(1, c.S):
                col = c.column(out, t, s, a)
                want_s = ident * scale_factor(c, c.scalers[s]).unsqueeze(1).float()
                rt = 1e-6 if c.dtype == torch.float32 else 2.0 ** -7
                torch.testing.assert_close(col[rows], want_s[rows], rtol=rt, atol=0)


@pytest.mark.parametrize("F,towers,dtype,bias,self_feat,sdeg,aggrs", [
    (12, 1, torch.float32, True, False, False, MIX), (16, 2, torch.float32, True, True, False, MIX),
    (10, 1, torch.float32, False, False, True, MIX), (40, 4, torch.float32, True, True, True, MIX),
    (16, 1, torch.bfloat16, True, False, False, MIX), (24, 3, torch.bfloat16, True, True, True, MIX),
    # with moments in the list: the families run one after the other on the same scratch
    (12, 1, torch.float32, True, False, False, ("softmin", "moment3", "softmax", "normalised_mean", "moment5"))])
def test_forward_matches_the_c_oracle_and_the_bar(emu, F, towers, dtype, bias, self_feat, sdeg, aggrs):
    c = Case(emu, 60, 400, F, seed=F + towers, dtype=dtype, towers=towers, bias=bias, self_feat=self_feat, sdeg=sdeg,
             scalers=SCALERS, aggrs=aggrs)
    assert c.hub_info.size(0) >= 1 and (c.deg == 0).sum() >= 5 and (c.deg == 1).sum() >= 4
    out = c.forward()
    rows = torch.ones(c.n, dtype=torch.bool)
    check_forward(c, out, rows)
    for a, name in enumerate(c.aggrs):
        for t in range(towers):
            for s in range(c.S):
                col = c.column(out, t, s, a)
                if name in WEIGHTED:         # rows without neighbours: 0, for every scaler
                    assert torch.equal(col[c.deg == 0], torch.zeros_like(col[c.deg == 0]))
                elif not name.startswith("moment"):   # the stubbed main path wrote nothing
                    assert torch.isnan(col).all()
    if self_feat:
        blocks = out.float().view(c.n, towers, -1)[:, :, :c.Ft]
        assert torch.isnan(blocks).all()
    assert same_bits(c.forward(), out)                                     # same bits on every run


def test_split_row_with_more_than_512_chunks(emu):
    c = Case(emu, 40, 150, 4, seed=3, big=40, huge=CHUNK * 520 + 3, aggrs=WEIGHTED, scalers=("identity",))
    assert int(c.hub_info[:, 2].max()) > 512
    out = c.forward()
    check_forward(c, out, torch.ones(c.n, dtype=torch.bool))
    assert same_bits(c.forward(), out)


def test_large_messages_stay_finite_and_within_the_bar(emu):
    """|m| up to 1e3: the reference's unshifted exp overflows to inf / inf = NaN here; the shifted form does not."""
    c = Case(emu, 60, 400, 8, seed=12, aggrs=WEIGHTED, scalers=("identity",))
    c.x = c.x * 300.0
    assert float(c.messages().abs().max()) > 1e3 * 0.9
    out = c.forward()
    assert torch.isfinite(out).all()
    check_forward(c, out, torch.ones(c.n, dtype=torch.bool))


def test_row_selection_skip_light_skip_hubs_and_masked_view(emu):
    c = Case(emu, 60, 400, 12, seed=8, aggrs=MIX)
    light, hub = c.deg < SPLIT, c.deg >= SPLIT
    cols = torch.zeros(c.W, dtype=torch.bool)
    for a, name in enumerate(c.aggrs):
        if name in WEIGHTED:
            for s in range(c.S):
                cols[(s * c.A + a) * c.Ft:(s * c.A + a + 1) * c.Ft] = True
    for flags, rows in ((_lib.FLAG_SKIP_LIGHT, hub), (_lib.FLAG_SKIP_HUBS, light)):
        out = c.forward(flags)
        check_forward(c, out, rows)
        assert torch.isnan(out[~rows]).all()
        assert torch.isfinite(out[rows][:, cols]).all()
    mask = torch.arange(c.n) % 2 == 0
    out = c.forward(view_mask=mask)
    sel = (mask & light) | hub
    check_forward(c, out, sel)
    assert torch.isnan(out[~sel]).all()


# ---- backward ----------------------------------------------------------------------------------------------------------
def run_bwd(c: Case, go, slots, f0=0, fc=None, per_slot=True):
    """slots: pna_aggregate_bwd_slots into [E, fc]; otherwise pna_aggregate_bwd, with col == NULL over the materialised
    messages when `per_slot` (one gradient row per slot), else through col into [n, F]."""
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
    xm = c.x[c.col.long()].contiguous()
    if per_slot:
        gg = torch.full((E, c.F), 0.5)
        d.gathered, d.col = xm.data_ptr(), None
    else:
        gg = torch.full((c.n, c.F), 0.5)
    rc = c.emu.pna_aggregate_bwd(C.byref(d), go.data_ptr(), c.W, gg.data_ptr(), c.F, None if gb is None else gb.data_ptr(),
                                 c.F, None)
    assert rc == 0, c.emu.emu_last_error()
    del xm
    return gg, gb


def upstream(c: Case, go_f, t, name):
    """(G, Gabs) [n, Ft]: the gradient of y summed over the positions of `name` and the scalers (identity, attenuation)."""
    d = c.deg.float()
    lg = torch.log(d + 1)
    att = torch.where(d > 0, c.avg["log"] / lg, torch.ones_like(lg)).unsqueeze(1)
    G, Gabs = 0, 0
    for a, nm in enumerate(c.aggrs):
        if nm == name:
            g0, g1 = c.column(go_f, t, 0, a), att * c.column(go_f, t, 1, a)
            G, Gabs = G + g0 + g1, Gabs + g0.abs() + g1.abs()
    return G, Gabs


@pytest.mark.parametrize("F,towers,dtype,bias,aggrs", [
    (12, 1, torch.float32, True, ("softmax",)), (16, 2, torch.float32, False, ("softmin",)),
    (40, 4, torch.float32, True, ("softmin", "softmax")), (8, 1, torch.float32, True, ("softmax", "softmax")),
    (12, 1, torch.float32, True, ("normalised_mean",)), (16, 2, torch.float32, True, ("softmax", "normalised_mean", "softmin")),
    (16, 1, torch.bfloat16, True, ("softmax", "softmin")), (24, 3, torch.bfloat16, True, ("normalised_mean",))])
def test_backward_atomic_and_slots_agree_and_match_float64(emu, F, towers, dtype, bias, aggrs):
    """Weighted aggregators only: the existing kernels (run for real here) then store a zero gradient for every slot, so
    what the buffers hold afterwards is the weighted terms alone."""
    c = Case(emu, 60, 400, F, seed=20 + F, dtype=dtype, towers=towers, bias=bias, aggrs=aggrs, scalers=("identity", "attenuation"))
    go = torch.randn(c.n, c.W, generator=torch.Generator().manual_seed(F))
    gs, gb = run_bwd(c, go, slots=True)
    assert torch.equal(run_bwd(c, go, slots=True)[0], gs)       # the same bits on every run
    al = 4 if dtype == torch.float32 else 8
    if F > al:                                                  # slab = column slice of the full-width run
        gs2, _ = run_bwd(c, go, slots=True, f0=al, fc=min(al, F - al))
        assert torch.equal(gs2, gs[:, al:al + gs2.size(1)])
    if "normalised_mean" not in aggrs:
        ga, gba = run_bwd(c, go, slots=False)
        assert torch.equal(gs, ga)                              # the same value of every slot in both instances
        if bias:
            assert torch.equal(gb, gba)
    # the atomic instance through col: per source row, the slot terms in some order
    gc, gbc = run_bwd(c, go, slots=False, per_slot=False)
    want_c = torch.full((c.n, c.F), 0.5, dtype=torch.float64).index_add(0, c.col.long(), gs.double())
    assert (gc.double() - want_c).abs().max() <= 1e-5 * (1 + float(want_c.abs().max()))
    if bias:
        assert torch.equal(gbc, gb)
    # against float64 autograd, per slot
    msg = c.messages()
    order = torch.sort(c.dst, stable=True).indices
    go_f = go.to(dtype).float()
    for t in range(towers):
        sl = slice(t * c.Ft, (t + 1) * c.Ft)
        g64 = torch.zeros(msg.size(0), c.Ft, dtype=torch.float64)
        tol = torch.zeros_like(g64)
        for name in sorted(set(aggrs)):
            G, Gabs = upstream(c, go_f, t, name)
            g, tl = WB.grad_bar(name, msg[:, sl], c.dst, c.n, G, Gabs, wsrc=c.src)
            g64, tol = g64 + g, tol + tl
        err = (gs[:, sl].double() - g64[order]).abs()
        lim = tol[order]
        assert (err <= lim).all(), float((err / lim).max())


def test_coef_row_ids_peer_and_col_null_refuse(emu):
    c = Case(emu, 30, 100, 8, seed=2, big=0, aggrs=("mean", "softmax"))
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
    assert emu.pna_aggregate_bwd(C.byref(d), go.data_ptr(), c.W, gg.data_ptr(), c.F, None, 0, None) == PNA_ERR_UNSUPPORTED
    # normalised_mean reads the source of every slot: col == NULL is refused, forward and backward
    c = Case(emu, 30, 100, 8, seed=2, big=0, aggrs=("normalised_mean",))
    out = torch.zeros(c.n, c.W)
    d = c.desc(out)
    d.col = None
    assert emu.pna_aggregate_fwd(C.byref(d), None) == PNA_ERR_UNSUPPORTED
    assert b"col" in emu.emu_last_error()
    d = c.desc(scratch_rows=6)
    d.col = None
    gs = torch.zeros(c.col.numel(), c.F)
    assert emu.pna_aggregate_bwd_slots(C.byref(d), go.data_ptr(), c.W, 0, c.F, gs.data_ptr(), c.F, None, 0, None) == \
        PNA_ERR_UNSUPPORTED
    assert torch.equal(out, torch.zeros_like(out))


def test_sources_outside_the_rows_get_weight_zero(emu):
    """A C caller that breaks the square-graph rule (col entries >= n_rows) reads no degree out of bounds: weight 0."""
    c = Case(emu, 40, 200, 8, seed=5, big=0, aggrs=("normalised_mean",), scalers=("identity",))
    x_big = torch.randn(c.n + 10, c.F, generator=torch.Generator().manual_seed(1))
    col = c.col.clone()
    col[::3] = c.n + 5
    c.x, c.col = x_big, col.contiguous()
    out = c.forward()
    src = c.src.clone()
    order = torch.sort(c.dst, stable=True).indices
    src[order] = col.long()
    c.src = src
    want = WO.weighted(c.messages(), c.dst, c.n, "normalised_mean", wsrc=src)
    light = c.deg < SPLIT
    assert torch.equal(c.column(out, 0, 0, 0)[light], want[light])
