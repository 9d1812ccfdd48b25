"""The slot-weight kernels (csrc/pna_aggregate_adj_weight.cuh, their backward in pna_aggregate_bwd.cu) executed on the HOST,
thread by thread (tests/emu), through the real C entry points pna_aggregate_fwd_weighted / _bwd_weighted / _bwd_slots_weighted.
A weighted call runs these kernels only, so every column they do not write keeps its NaN.  Every row -- light, split, and one
split row with more than 512 chunks -- must equal a scalar restatement of the rounding order (numpy float32, one rounding per
operation, split rows merged in chunk order) bit for bit; with all-ones weights the light rows must equal the C oracle's
unweighted values bit for bit."""
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from oracle import c_oracle
from pna_b200 import _lib
from test_moments_emulated import CHUNK, SPLIT, Case, _STUBS, same_bits

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")

HERE = os.path.dirname(os.path.abspath(__file__))
SIX = ("sum", "mean", "min", "max", "var", "std")
f32 = np.float32


def _build():
    import importlib.util
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(HERE, "emu", "build_emu.py"))
    be = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(be)
    srcs = [os.path.join(be.CSRC, n) for n in ("pna_aggregate.cu", "pna_aggregate_bwd.cu")]
    deps = srcs + [os.path.join(be.CSRC, n) for n in ("pna_aggregate.cuh", "pna_aggregate_moments.cuh", "pna_aggregate_weighted.cuh",
                                                      "pna_aggregate_adj_weight.cuh", "common.cuh")] + [
        os.path.join(be.HERE, "cuda_host_shim.h"), os.path.join(be.ROOT, "include", "pna_b200.h"), __file__]
    os.makedirs(be.BUILD, exist_ok=True)
    lib = os.path.join(be.BUILD, "libadj_weight_emu.so")
    if os.path.exists(lib) and all(os.path.getmtime(lib) >= os.path.getmtime(d) for d in deps):
        return lib
    body = ""
    for s in srcs:
        t = be.strip_inline_ptx(be.rewrite_launches(open(s).read()))
        body += re.sub(r'#include "(pna_aggregate\.cuh|common\.cuh)"', lambda m: f'#include "{be.CSRC}/{m.group(1)}"', t) + "\n"
    tu = os.path.join(be.BUILD, "adj_weight_emu.cpp")
    with open(tu, "w") as f:
        f.write(f'#include "{be.HERE}/cuda_host_shim.h"\n#include <stdarg.h>\n#include <stdio.h>\n')
        f.write(body)
        f.write(_STUBS)
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    subprocess.run(["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-w", f"-I{cuda_inc}", tu, "-o", lib],
                   check=True)
    return lib


@pytest.fixture(scope="module")
def emu():
    try:
        L = C.CDLL(_build())
    except Exception as exc:            # no CUDA headers on this machine
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    ws = [C.POINTER(_lib.AggStruct), C.c_void_p, C.c_void_p]
    L.pna_aggregate_fwd_weighted.argtypes = ws + [C.c_void_p]
    L.pna_aggregate_bwd_weighted.argtypes = ws + [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    L.pna_aggregate_bwd_slots_weighted.argtypes = ws + [C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int64,
                                                        C.c_void_p, C.c_int64, C.c_void_p]
    return L


def weights(c: Case, kind, seed=0):
    """[E] fp32 slot weights in CSR order."""
    E = c.col.numel()
    g = torch.Generator().manual_seed(seed)
    if kind == "ones":
        return torch.ones(E)
    w = torch.rand(E, generator=g) * 1.75 + 0.25
    if kind == "signed":                # negative and zero entries: in the sums, not in min / max
        w[torch.rand(E, generator=g) < 0.15] *= -1
        w[torch.rand(E, generator=g) < 0.05] = 0
    return w.contiguous()


def run_fwd(c: Case, w, flags=0, in_order=False):
    out = torch.full((c.n, c.W), float("nan")).to(c.dtype)
    d = c.desc(out, flags)
    keep = None
    if in_order:                        # messages already in CSR order (col == NULL)
        keep = c.x[c.col.long()].contiguous()
        d.gathered, d.col = keep.data_ptr(), None
    rc = c.emu.pna_aggregate_fwd_weighted(C.byref(d), w.data_ptr(), None, None)
    assert rc == 0, c.emu.emu_last_error()
    del keep
    return out


# ---- the scalar restatement -------------------------------------------------------------------------------------------
def slot_messages(c: Case):
    """[E, F] float32 numpy messages in CSR slot order, as the kernel forms them (gathered row + row_bias)."""
    x = c.x.float()[c.col.long()]
    if c.bias is not None:
        dst = torch.repeat_interleave(torch.arange(c.n), c.deg)
        x = x + c.bias.float()[dst]
    return x.numpy().astype(f32)


def row_stats(m, w, beg, end):
    """S, Q, min, max over slots [beg, end) per chunk, merged in chunk order (one chunk for light rows); W in slot order."""
    deg = end - beg
    bounds = [(beg, end)] if deg < SPLIT else [(b, min(b + CHUNK, end)) for b in range(beg, end, CHUNK)]
    F = m.shape[1]
    S, Q = np.zeros(F, f32), np.zeros(F, f32)
    mn, mx = np.full(F, np.inf, f32), np.full(F, -np.inf, f32)
    for b, e in bounds:
        s, q = np.zeros(F, f32), np.zeros(F, f32)
        for k in range(b, e):
            s = s + m[k] * w[k]
            q = q + (m[k] * m[k]) * w[k]
            if w[k] > 0:
                mn, mx = np.minimum(mn, m[k]), np.maximum(mx, m[k])
        S, Q = S + s, Q + q
    W = f32(0)
    for k in range(beg, end):
        W = f32(W + w[k])
    return S, Q, mn, mx, W


def restate_forward(c: Case, w, relu_var=False):
    """{aggregator: [n, F]} unscaled."""
    m, w = slot_messages(c), w.numpy().astype(f32)
    rp = c.rowptr.tolist()
    res = {a: np.zeros((c.n, c.F), f32) for a in SIX}
    with np.errstate(all="ignore"):
        for r in range(c.n):
            if rp[r + 1] == rp[r]:
                res["std"][r] = np.sqrt(f32(0) + f32(1e-5))
                continue
            S, Q, mn, mx, W = row_stats(m, w, rp[r], rp[r + 1])
            mean = S / W
            var = Q / W - mean * mean
            none = mx < mn
            res["sum"][r], res["mean"][r] = S, mean
            res["min"][r], res["max"][r] = np.where(none, f32(0), mn), np.where(none, f32(0), mx)
            res["var"][r] = np.fmax(var, f32(0)) if relu_var else var          # fmax: fmaxf's NaN rule
            res["std"][r] = np.sqrt(np.fmax(var, f32(0)) + f32(1e-5))
    return res


def bits_equal(a, b):
    return np.array_equal(np.asarray(a, f32).view(np.int32), np.asarray(b, f32).view(np.int32))


@pytest.mark.parametrize("F,towers,dtype,bias,self_feat,kind,in_order", [
    (8, 1, torch.float32, True, False, "pos", False), (12, 2, torch.float32, True, True, "signed", False),
    (10, 1, torch.float32, False, False, "signed", True), (16, 2, torch.bfloat16, True, True, "signed", False),
    (8, 1, torch.bfloat16, True, False, "pos", True)])
def test_forward_matches_the_restatement_bit_for_bit(emu, F, towers, dtype, bias, self_feat, kind, in_order):
    c = Case(emu, 60, 400, F, seed=F + towers, dtype=dtype, towers=towers, bias=bias, self_feat=self_feat, aggrs=SIX,
             scalers=("identity", "amplification", "inverse_linear"))
    assert c.hub_info.size(0) >= 1 and (c.deg == 0).sum() >= 5
    w = weights(c, kind, seed=F)
    out = run_fwd(c, w, in_order=in_order)
    want = restate_forward(c, w)
    for a, name in enumerate(SIX):
        for t in range(towers):
            got = c.column(out, t, 0, a).numpy()
            ref = want[name][:, t * c.Ft:(t + 1) * c.Ft]
            if dtype == torch.bfloat16:
                ref = torch.from_numpy(ref).to(torch.bfloat16).float().numpy()
            assert bits_equal(got, ref), (name, t)
            for s in (1, 2):         # scaled columns: fl(y * factor) of the slot-count degree (no scaler degree given)
                D = c.deg.double()
                fac = torch.log(D + 1) / c.avg["log"] if s == 1 else torch.where(D > 0, c.avg["lin"] / D, torch.ones_like(D))
                torch.testing.assert_close(c.column(out, t, s, a).double(), c.column(out, t, 0, a).double() * fac.unsqueeze(1),
                                           rtol=1e-6 if dtype == torch.float32 else 2.0 ** -7, atol=0, equal_nan=True)
    if self_feat:
        blocks = out.float().view(c.n, towers, -1)[:, :, :c.Ft]
        assert torch.equal(blocks, c.self_feat.float().view(c.n, towers, c.Ft))
    assert same_bits(run_fwd(c, w, in_order=in_order), out)


def test_split_row_with_more_than_512_chunks_and_relu_var(emu):
    c = Case(emu, 40, 150, 4, seed=3, big=40, huge=CHUNK * 520 + 3, aggrs=SIX, scalers=("identity",))
    assert int(c.hub_info[:, 2].max()) > 512
    w = weights(c, "signed", seed=9)
    out = run_fwd(c, w, flags=_lib.FLAG_RELU_VAR)
    want = restate_forward(c, w, relu_var=True)
    for a, name in enumerate(SIX):
        assert bits_equal(c.column(out, 0, 0, a).numpy(), want[name]), name


def test_all_ones_weights_give_the_c_oracle_unweighted_bits_on_light_rows(emu):
    c = Case(emu, 60, 400, 12, seed=5, aggrs=SIX, scalers=("identity",))
    out = run_fwd(c, weights(c, "ones"))
    msg = c.messages()
    want = c_oracle.aggregate(msg, torch.stack([torch.arange(msg.size(0)), c.dst]), list(SIX), ["identity"], c.avg)[:c.n]
    light = c.deg < SPLIT
    for a in range(len(SIX)):
        assert torch.equal(c.column(out, 0, 0, a)[light], want[:, a * c.F:(a + 1) * c.F][light]), SIX[a]


def test_real_scaler_degree_and_zero_weight_rows(emu):
    """scaler_degree_f alone runs these kernels with every weight 1; a row whose weights sum to 0 gets the IEEE quotient."""
    c = Case(emu, 40, 200, 8, seed=7, big=0, aggrs=("mean", "sum", "max"), scalers=("identity", "linear"))
    D = (c.deg.float() * 0.75 + 0.5).contiguous()
    out = torch.full((c.n, c.W), float("nan"))
    d = c.desc(out)
    assert emu.pna_aggregate_fwd_weighted(C.byref(d), None, D.data_ptr(), None) == 0, emu.emu_last_error()
    plain = restate_forward(c, weights(c, "ones"))
    assert bits_equal(c.column(out, 0, 0, 0).numpy(), plain["mean"])
    torch.testing.assert_close(c.column(out, 0, 1, 1), c.column(out, 0, 0, 1) * (D / c.avg["lin"]).unsqueeze(1), rtol=1e-6, atol=0)
    w = weights(c, "pos")
    r = int((c.deg > 1).nonzero()[0])
    b, e = int(c.rowptr[r]), int(c.rowptr[r + 1])
    w[b:e] = 0
    w[b], w[b + 1] = 1.5, -1.5
    out = run_fwd(c, w)
    assert torch.isinf(c.column(out, 0, 0, 0)[r]).any() or torch.isnan(c.column(out, 0, 0, 0)[r]).any()
    assert bits_equal(c.column(out, 0, 0, 1).numpy()[r], restate_forward(c, w)["sum"][r])


# ---- backward ----------------------------------------------------------------------------------------------------------
def restate_slot_grads(c: Case, w, go, relu_var=False):
    """[E, F] per-slot gradients and [n, F] grad_row_bias, identity scaler only: the coefficients of the unweighted backward
    at cnt = W_i, then fl(w * fl(c0 + c1 m)) + the routed min / max terms."""
    m, wn = slot_messages(c), w.numpy().astype(f32)
    go = go.float().numpy().astype(f32)
    rp = c.rowptr.tolist()
    E = m.shape[0]
    gs, gb = np.zeros((E, c.F), f32), np.zeros((c.n, c.F), f32)
    with np.errstate(all="ignore"):
        for r in range(c.n):
            beg, end = rp[r], rp[r + 1]
            if beg == end:
                continue
            S, Q, mn, mx, W = row_stats(m, wn, beg, end)
            mean = S / W
            var = Q / W - mean * mean
            sd = np.sqrt(np.fmax(var, f32(0)) + f32(1e-5))
            c0, c1, gmin, gmax = (np.zeros(c.F, f32) for _ in range(4))
            for a, name in enumerate(c.aggrs):
                g = np.zeros(c.F, f32) + c.column(torch.from_numpy(go), 0, 0, a).numpy()[r]
                if name == "sum":
                    c0 = c0 + g
                elif name == "mean":
                    c0 = c0 + g / W
                elif name == "min":
                    gmin = gmin + g
                elif name == "max":
                    gmax = gmax + g
                else:
                    if name == "var":
                        t = (f32(2) * g) / W
                        if relu_var:
                            t = np.where(var > 0, t, f32(0))
                    else:
                        t = np.where(var > 0, g / (W * sd), f32(0))
                    c1 = c1 + t
                    c0 = c0 - t * mean
            # the first slot attaining the extremum among the positive weights (chunks merged in order: the same slot)
            amn, amx = np.full(c.F, -1), np.full(c.F, -1)
            cmn, cmx = np.full(c.F, np.inf, f32), np.full(c.F, -np.inf, f32)
            for k in range(beg, end):
                if wn[k] > 0:
                    lt, gt = m[k] < cmn, m[k] > cmx
                    cmn, amn = np.where(lt, m[k], cmn), np.where(lt, k, amn)
                    cmx, amx = np.where(gt, m[k], cmx), np.where(gt, k, amx)
            bounds = [(beg, end)] if end - beg < SPLIT else [(b, min(b + CHUNK, end)) for b in range(beg, end, CHUNK)]
            tot = np.zeros(c.F, f32)
            for b, e in bounds:
                share = np.zeros(c.F, f32)
                for k in range(b, e):
                    g = f32(0) + wn[k] * (c0 + c1 * m[k])
                    g = g + np.where(amn == k, gmin, f32(0))
                    g = g + np.where(amx == k, gmax, f32(0))
                    gs[k] = g
                    share = share + g
                tot = tot + share
            gb[r] = tot
    return gs, gb


def run_bwd(c: Case, w, go, slots):
    E = c.col.numel()
    d = c.desc(scratch_rows=6)
    gb = torch.full((c.n, c.F), 0.25) if c.bias is not None else None
    go = go.to(c.dtype).contiguous()
    if slots:
        gs = torch.full((E, c.F), 0.5)
        rc = c.emu.pna_aggregate_bwd_slots_weighted(C.byref(d), w.data_ptr(), None, go.data_ptr(), c.W, 0, c.F, gs.data_ptr(), c.F,
                                                    None if gb is None else gb.data_ptr(), c.F, None)
    else:
        gs = torch.zeros((c.n, c.F))
        rc = c.emu.pna_aggregate_bwd_weighted(C.byref(d), w.data_ptr(), None, go.data_ptr(), c.W, gs.data_ptr(), c.F,
                                              None if gb is None else gb.data_ptr(), c.F, None)
    assert rc == 0, c.emu.emu_last_error()
    return gs, gb


@pytest.mark.parametrize("F,dtype,bias,kind,aggrs", [
    (8, torch.float32, True, "signed", SIX), (12, torch.float32, False, "pos", ("mean", "std", "max")),
    (8, torch.bfloat16, True, "signed", ("sum", "var", "min", "mean")), (4, torch.float32, True, "ones", SIX)])
def test_backward_matches_the_restatement_bit_for_bit(emu, F, dtype, bias, kind, aggrs):
    c = Case(emu, 60, 400, F, seed=30 + F, dtype=dtype, bias=bias, aggrs=aggrs, scalers=("identity",))
    assert c.hub_info.size(0) >= 1
    w = weights(c, kind, seed=F)
    go = torch.randn(c.n, c.W, generator=torch.Generator().manual_seed(F))
    gs, gb = run_bwd(c, w, go, slots=True)
    want_s, want_b = restate_slot_grads(c, w, go.to(dtype))
    assert bits_equal(gs.numpy(), want_s)
    if bias:
        assert bits_equal(gb.numpy(), want_b)
    assert torch.equal(run_bwd(c, w, go, slots=True)[0], gs)
    # the atomic instance adds the same slot values into grad_gathered[col[s]]
    gg, gba = run_bwd(c, w, go, slots=False)
    want_g = torch.zeros(c.n, c.F, dtype=torch.float64).index_add(0, c.col.long(), gs.double())
    assert (gg.double() - want_g).abs().max() <= 1e-5 * (1 + float(want_g.abs().max()))
    if bias:
        assert torch.equal(gba, gb)


def test_all_ones_backward_equals_the_unweighted_restatement(emu):
    """w = 1: W_i = d, fl(1 * x) = x -- the per-slot values of the unweighted coefficients."""
    c = Case(emu, 60, 400, 8, seed=41, aggrs=SIX, scalers=("identity",), big=0)
    go = torch.randn(c.n, c.W, generator=torch.Generator().manual_seed(2))
    gs, _ = run_bwd(c, weights(c, "ones"), go, slots=True)
    want, _ = restate_slot_grads(c, torch.ones(c.col.numel()), go)
    assert bits_equal(gs.numpy(), want)
