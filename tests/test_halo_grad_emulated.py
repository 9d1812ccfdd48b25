"""The pull plane's backward on the HOST: pna_halo_grad_pull (csrc/pna_peer.cu) executed thread by thread (tests/emu) for W
"ranks" in one process, on the reverse plans pna_b200/dist.py builds from real pull plans.  The gradient return must equal a
sequential loop doing the same fp32 adds in the same order, bit for bit, and touch nothing else; and the oracle's autograd
on every rank's [local ; halo], followed by the gradient return, must give the oracle's autograd over the whole graph."""
import ctypes as C
import importlib.util
import os
import shutil

import pytest
import torch

from oracle import pna_oracle as O
from pna_b200 import dist as pd

pytestmark = pytest.mark.skipif(shutil.which("g++") is None, reason="needs g++")
A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]


@pytest.fixture(scope="module")
def emu():
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu", "build_emu.py"))
    build_emu = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(build_emu)
    try:
        L = C.CDLL(build_emu.build("pna_peer.cu"))
    except Exception as exc:
        pytest.skip(f"emulation library did not build: {exc}")
    L.emu_last_error.restype = C.c_char_p
    L.pna_halo_grad_pull.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int64, C.c_void_p,
                                     C.c_int64, C.c_int32, C.c_void_p]
    return L


def partitioned(n, e, world, seed, hub=0):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, int(n * 0.9), (e,), generator=g)
    if hub:                                       # one destination far above the split threshold
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.full((hub,), n // 3)])
    deg = torch.bincount(dst, minlength=n)
    bounds = pd.partition_bounds(deg, world)
    plans = []
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        mine = (dst >= lo) & (dst < hi)
        plans.append(pd.build_pull_plan(src[mine], dst[mine], bounds, r, world))
    return src, dst, deg, bounds, plans


def grad_pull(emu, table, ld, gp, grad, f):
    rc = emu.pna_halo_grad_pull(table.data_ptr(), ld, gp.rows.data_ptr(), gp.rowptr.data_ptr(), gp.enc.data_ptr(), gp.shift,
                                gp.n_rows, grad.data_ptr(), grad.stride(0), f, None)
    assert rc == 0, emu.emu_last_error()


def tail_table(bufs, plans, ld):
    return torch.tensor([b.data_ptr() + p.n_local * ld * 4 for b, p in zip(bufs, plans)], dtype=torch.int64)


@pytest.mark.parametrize("world,f,pitch_pad", [(2, 8, 0), (3, 75, 0), (4, 128, 0), (4, 256, 0), (2, 520, 0), (8, 8, 4),
                                               (3, 128, 4), (4, 75, 5), (2, 256, 3), (8, 520, 4)])
def test_emulated_grad_pull_is_the_sequential_sum(emu, world, f, pitch_pad):
    n, e = 90 * world, 700 * world
    _, _, _, bounds, plans = partitioned(n, e, world, seed=world * 100 + f)
    gplans = pd.grad_return_plans(plans)
    # the reverse plans list exactly the (owner row, peer, halo position) triples of the pull plans, peers ascending per row
    for r, gp in enumerate(gplans):
        mask = (1 << gp.shift) - 1
        got = set()
        for i in range(gp.n_rows):
            peers = [int(v) >> gp.shift for v in gp.enc[int(gp.rowptr[i]):int(gp.rowptr[i + 1])]]
            assert peers == sorted(peers) and len(set(peers)) == len(peers)
            for v in gp.enc[int(gp.rowptr[i]):int(gp.rowptr[i + 1])].tolist():
                got.add((int(gp.rows[i]), v >> gp.shift, v & mask))
        lo = int(bounds[r])
        want = {(int(h) - lo, p, i) for p, pl in enumerate(plans) for i, h in enumerate(pl.halo_ids.tolist())
                if int(bounds[r]) <= h < int(bounds[r + 1])}
        assert got == want
        assert gp.peer_n_local == [p.n_local for p in plans]
    assert sum(gp.n_rows for gp in gplans) > 0
    ld = f + pitch_pad
    rows = max(p.n_local + p.n_halo for p in plans)
    g = torch.Generator().manual_seed(f)
    bufs = [torch.randn((rows + 2, ld), generator=g) for _ in range(world)]     # every rank's fp32 gradient buffer
    before = [b.clone() for b in bufs]
    table = tail_table(bufs, plans, ld)
    for r, (p, gp) in enumerate(zip(plans, gplans)):
        grad = torch.randn((p.n_local + 3, ld), generator=g)                      # 3 rows past the rank's rows: untouched
        want = grad.clone()
        mask = (1 << gp.shift) - 1
        for i in range(gp.n_rows):
            row = int(gp.rows[i])
            for v in gp.enc[int(gp.rowptr[i]):int(gp.rowptr[i + 1])].tolist():
                q = v >> gp.shift
                want[row, :f] = want[row, :f] + bufs[q][plans[q].n_local + (v & mask), :f]
        grad_pull(emu, table, ld, gp, grad, f)
        assert torch.equal(grad, want), f"rank {r}"
        touched = torch.zeros(grad.size(0), dtype=torch.bool)
        touched[gp.rows.long()] = True
        assert torch.equal(grad[~touched], want[~touched])                         # rows without contributions
    for b, b0 in zip(bufs, before):
        assert torch.equal(b, b0)                                                 # the peers' buffers are only read


def test_emulated_grad_pull_empty_and_bad_arguments(emu):
    one = torch.zeros(4, dtype=torch.int32)
    g = torch.zeros(2, 8)
    assert emu.pna_halo_grad_pull(None, 8, None, None, None, 4, 0, None, 8, 8, None) == 0        # nothing to do
    assert emu.pna_halo_grad_pull(None, 8, one.data_ptr(), one.data_ptr(), one.data_ptr(), 4, 1, g.data_ptr(), 8, 8, None) == -1
    assert emu.pna_halo_grad_pull(one.data_ptr(), 8, one.data_ptr(), one.data_ptr(), one.data_ptr(), 0, 1, g.data_ptr(), 8, 8, None) == -1
    assert emu.pna_halo_grad_pull(one.data_ptr(), 8, one.data_ptr(), one.data_ptr(), one.data_ptr(), 31, 1, g.data_ptr(), 8, 8, None) == -1
    assert emu.pna_halo_grad_pull(one.data_ptr(), 4, one.data_ptr(), one.data_ptr(), one.data_ptr(), 4, 1, g.data_ptr(), 8, 8, None) == -1
    assert emu.pna_halo_grad_pull(one.data_ptr(), 8, one.data_ptr(), one.data_ptr(), one.data_ptr(), 4, -1, g.data_ptr(), 8, 8, None) == -1


@pytest.mark.parametrize("world,f,hub", [(2, 12, 600), (3, 8, 900), (4, 16, 0)])
def test_host_gradient_return_gives_the_whole_graph_gradient(emu, world, f, hub):
    n, e = 240, 2400
    src, dst, deg, bounds, plans = partitioned(n, e, world, seed=7 + world, hub=hub)
    gplans = pd.grad_return_plans(plans)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(n, f, generator=g)
    avg = O.avg_deg_from_histogram(torch.bincount(deg))
    w = torch.randn(n, len(A4) * len(S3) * f, generator=g)
    xr = x.clone().requires_grad_(True)
    (O.simple_propagate(xr, torch.stack([src, dst]), A4, S3, avg) * w).sum().backward()
    rows = max(p.n_local + p.n_halo for p in plans)
    bufs = [torch.full((rows, f), float("nan")) for _ in range(world)]
    grads = []
    for r, p in enumerate(plans):                     # every rank: autograd on [local ; halo], stage the halo rows' gradient
        ext = torch.cat([x[p.lo:p.hi], x[p.halo_ids]]).requires_grad_(True)
        out = O.simple_propagate(ext, torch.stack([p.src_ext, p.dst_local]), A4, S3, avg)[: p.n_local]
        (out * w[p.lo:p.hi]).sum().backward()
        bufs[r][p.n_local:p.n_local + p.n_halo] = ext.grad[p.n_local:]
        grads.append(ext.grad[: p.n_local].clone())
    table = tail_table(bufs, plans, f)
    for r in range(world):                            # every owner: pull and add
        grad_pull(emu, table, f, gplans[r], grads[r], f)
    got = torch.cat(grads)
    assert sum(p.n_halo for p in plans) > 0
    # the same per-edge terms, summed per rank and then across ranks: fp32 reordering only
    torch.testing.assert_close(got, xr.grad, rtol=1e-5, atol=1e-5 * float(xr.grad.abs().max()))


def test_grad_return_shift_rejects_overflow():
    assert pd.grad_return_shift(1, 8) == 1 and pd.grad_return_shift(1025, 2) == 11
    with pytest.raises(ValueError):
        pd.grad_return_shift(1 << 29, 8)               # 8 << 29 = 2^32
    with pytest.raises(ValueError):
        pd.grad_return_shift((1 << 30) + 1, 2)         # 31 bits
