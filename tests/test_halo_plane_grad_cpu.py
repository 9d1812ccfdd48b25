"""The halo plane's backward on the CPU.  The owner's reverse plan (``dist.halo_grad_return_plan``) is checked against what
the transposed all-to-all delivers: on halo plans of W ranks built in one process (one thread per rank), and through gloo
with world 2 and 3.  The gradient return itself is pna_halo_grad_pull (csrc/pna_peer.cu) run thread by thread (tests/emu)
with a pointer table that aliases one receive buffer: it must equal a sequential loop bit for bit and, behind the oracle's
autograd on every rank's [local ; halo], give the oracle's autograd over the whole graph."""
import ctypes as C
import importlib.util
import os
import shutil
import socket
import sys
import threading
from unittest import mock

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import pna_oracle as O
from pna_b200 import dist as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]


# ---- W ranks in one process --------------------------------------------------------------------------------------------
class ThreadedAllToAll:
    """``torch.distributed.all_to_all_single`` among W threads of one process; the caller's rank is passed as ``group``.
    CUDA inputs are complete (stream synchronised) before any peer reads them, and every peer has read them before any
    rank returns and may overwrite them."""

    def __init__(self, world: int):
        self.world = world
        self.bar = threading.Barrier(world, timeout=120)
        self.slots = [None] * world
        self.calls = 0

    def abort(self):
        self.bar.abort()

    def __call__(self, output, input, output_split_sizes=None, input_split_sizes=None, group=None, async_op=False):
        r, w = int(group), self.world
        assert output.dtype == input.dtype and output.is_contiguous() and input.is_contiguous() and not async_op
        ins = list(input_split_sizes) if input_split_sizes is not None else [input.size(0) // w] * w
        outs = list(output_split_sizes) if output_split_sizes is not None else [output.size(0) // w] * w
        assert sum(ins) == input.size(0) and sum(outs) == output.size(0)
        if input.is_cuda:
            torch.cuda.current_stream(input.device).synchronize()
        self.slots[r] = (input, ins)
        if r == 0:
            self.calls += 1
        self.bar.wait()
        o = 0
        for q in range(w):
            t, s = self.slots[q]
            a = sum(s[:r])
            assert s[r] == outs[q], f"rank {q} sends {s[r]} rows to rank {r}, which expects {outs[q]}"
            output[o:o + s[r]].copy_(t[a:a + s[r]])
            o += s[r]
        if output.is_cuda:
            torch.cuda.current_stream(output.device).synchronize()
        self.bar.wait()


def run_ranks(world, fn, abort=()):
    """fn(r) on one thread per rank; the first error aborts the barriers in ``abort`` so the other ranks stop too."""
    out, errors = [None] * world, []

    def main(r):
        try:
            out[r] = fn(r)
        except BaseException as exc:  # noqa: BLE001 -- reported below; the other ranks are released
            errors.append((r, exc))
            for a in abort:
                a()
    threads = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads)
    assert not errors, errors
    return out


def partitioned_graph(n, e, world, seed, hub=0, local_head=False):
    """Random multigraph cut into `world` destination ranges.  ``hub``: extra in-edges of one row (a split row);
    ``local_head``: the first quarter's rows take their sources from the first quarter only, so the ranks there need
    nothing from the ranks behind them (empty segments)."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, int(n * 0.9), (e,), generator=g)
    if hub:
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.full((hub,), n // 3)])
    if local_head:
        head = dst < n // 4
        src[head] = torch.randint(0, n // 4, (int(head.sum()),), generator=g)
    deg = torch.bincount(dst, minlength=n)
    return src, dst, deg, pd.partition_bounds(deg, world)


def halo_plans(src, dst, bounds, world):
    """Every rank's HaloPlan (build_halo_plan with its collectives), W threads of one process."""
    a2a = ThreadedAllToAll(world)

    def plan(r):
        mine = (dst >= bounds[r]) & (dst < bounds[r + 1])
        return pd.build_halo_plan(src[mine], dst[mine], bounds, r, world, group=r)
    with mock.patch.object(pd.dist, "all_to_all_single", a2a):
        return run_ranks(world, plan, abort=[a2a.abort])


def _offsets(splits):
    out, o = [], 0
    for s in splits:
        out.append(o)
        o += s
    return out


def reverse_all_to_all(plans, halo_rows):
    """What every owner receives in the backward: from each peer p, in peer order, p's rows of that owner's segment."""
    world = len(plans)
    recv = []
    for r in range(world):
        parts = []
        for p in range(world):
            o = _offsets(plans[p].recv_splits)[r]
            parts.append(halo_rows[p][o:o + plans[p].recv_splits[r]])
        recv.append(torch.cat(parts))
    return recv


def check_reverse_plan(plans, r, received_ids):
    """received_ids[k]: global id of the row whose gradient arrives at position k of owner r's receive buffer."""
    p_r = plans[r]
    gp = pd.halo_grad_return_plan(p_r)
    assert (gp.rank, gp.world) == (r, p_r.world) and gp.peer_n_local is None
    assert (p_r.world << gp.shift) < 2 ** 31
    assert gp.shift == pd.grad_return_shift(max(p_r.send_splits), p_r.world)
    mask, send_off = (1 << gp.shift) - 1, _offsets(p_r.send_splits)
    rows = gp.rows.tolist()
    assert rows == sorted(set(rows))                                      # no row repeats
    assert int(gp.rowptr[0]) == 0 and int(gp.rowptr[-1]) == gp.enc.numel() and gp.rowptr.dtype == torch.int32
    named = []
    for i, row in enumerate(rows):
        slots = gp.enc[int(gp.rowptr[i]):int(gp.rowptr[i + 1])].tolist()
        assert slots, "a listed row has no slot"
        peers = [v >> gp.shift for v in slots]
        assert peers == sorted(set(peers))                                # ascending peer rank, each peer once
        for v in slots:
            peer, q = v >> gp.shift, v & mask
            assert peer != r and q < p_r.send_splits[peer]
            k = send_off[peer] + q
            assert int(received_ids[k]) == p_r.lo + row, (r, row, peer, q)
            named.append(k)
    assert sorted(named) == list(range(int(p_r.send_idx.numel())))      # every receive position exactly once
    return gp


@pytest.mark.parametrize("world,hub,local_head", [(2, 0, False), (2, 500, True), (3, 700, False), (4, 0, True),
                                                  (5, 900, False), (6, 300, True), (7, 0, False), (8, 1200, True)])
def test_halo_reverse_plan_names_every_receive_position(world, hub, local_head):
    n = 80 * world
    src, dst, _, bounds = partitioned_graph(n, 600 * world, world, seed=world * 31 + hub, hub=hub, local_head=local_head)
    plans = halo_plans(src, dst, bounds, world)
    for p in plans:                                   # the threaded builder against the halo it describes
        assert p.halo_ids.numel() == p.n_halo and sum(p.recv_splits) == p.n_halo
    received = reverse_all_to_all(plans, [p.halo_ids for p in plans])
    gps = [check_reverse_plan(plans, r, received[r]) for r in range(world)]
    assert sum(gp.n_rows for gp in gps) > 0
    empty = [(r, q) for r in range(world) for q in range(world) if q != r and plans[r].send_splits[q] == 0]
    if local_head and world >= 4:
        assert empty                                  # some owner sends nothing to some peer: empty segments are covered


def test_halo_reverse_plan_of_a_rank_without_peers():
    src, dst, _, bounds = partitioned_graph(200, 1500, 2, seed=4)
    plan = halo_plans(src, dst, bounds, 2)[0]
    lone = pd.HaloPlan(0, 1, 0, plan.n_local, plan.n_local, 0, plan.src_ext, plan.dst_local, plan.halo_ids[:0], [0], [0],
                       plan.send_idx[:0], plan.interior)
    gp = pd.halo_grad_return_plan(lone)
    assert gp.n_rows == 0 and gp.rowptr.tolist() == [0] and gp.enc.numel() == 0


# ---- gloo: the real collectives ----------------------------------------------------------------------------------------
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _gloo_worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from pna_b200 import dist as pdist
        src, dst, _, bounds = partitioned_graph(300, 3000, world, seed=17, hub=400)
        mine = (dst >= bounds[rank]) & (dst < bounds[rank + 1])
        plan = pdist.build_halo_plan(src[mine], dst[mine], bounds, rank, world)
        # every halo row, tagged with its global id and the rank that holds the copy, back to its owner with the real split
        # sizes of the backward (the forward's swapped)
        tags = torch.stack([plan.halo_ids, torch.full_like(plan.halo_ids, rank)], 1)
        recv = torch.empty((int(plan.send_idx.numel()), 2), dtype=torch.int64)
        dist.all_to_all_single(recv, tags, output_split_sizes=plan.send_splits, input_split_sizes=plan.recv_splits)
        gp = pdist.halo_grad_return_plan(plan)
        mask, send_off = (1 << gp.shift) - 1, _offsets(plan.send_splits)
        seen = []
        for i in range(gp.n_rows):
            for v in gp.enc[int(gp.rowptr[i]):int(gp.rowptr[i + 1])].tolist():
                k = send_off[v >> gp.shift] + (v & mask)
                assert recv[k].tolist() == [plan.lo + int(gp.rows[i]), v >> gp.shift], (k, recv[k].tolist())
                seen.append(k)
        assert sorted(seen) == list(range(recv.size(0)))
        q.put((rank, "ok", gp.n_rows))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), 0))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_halo_reverse_plan_matches_the_gloo_all_to_all(world):
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for r in res:
        assert r[1] == "ok", r[1]
    assert all(r[2] > 0 for r in res)                 # every rank has rows held by a peer


# ---- the gradient return, emulated ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu():
    if shutil.which("g++") is None:
        pytest.skip("needs g++")
    spec = importlib.util.spec_from_file_location("build_emu", os.path.join(ROOT, "tests", "emu", "build_emu.py"))
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


def return_grad(emu, plan, gp, recv, grad, f):
    """Owner side of the backward: the table aims every peer's slot at its segment of the one receive buffer."""
    ld = recv.stride(0)
    table = torch.tensor([recv.data_ptr() + o * ld * 4 for o in _offsets(plan.send_splits)], dtype=torch.int64)
    rc = emu.pna_halo_grad_pull(table.data_ptr(), ld, gp.rows.data_ptr(), gp.rowptr.data_ptr(), gp.enc.data_ptr(), gp.shift,
                                gp.n_rows, grad.data_ptr(), grad.stride(0), f, None)
    assert rc == 0, emu.emu_last_error()


@pytest.mark.parametrize("world,f,pitch_pad,hub,local_head", [(2, 8, 0, 0, False), (3, 75, 0, 600, True), (4, 128, 0, 0, False),
                                                              (4, 256, 3, 900, True), (8, 8, 4, 0, True), (5, 520, 4, 700, False)])
def test_emulated_halo_grad_return_is_the_sequential_sum(emu, world, f, pitch_pad, hub, local_head):
    n = 90 * world
    src, dst, _, bounds = partitioned_graph(n, 700 * world, world, seed=world * 100 + f, hub=hub, local_head=local_head)
    plans = halo_plans(src, dst, bounds, world)
    ld = f + pitch_pad
    g = torch.Generator().manual_seed(f)
    halo_grads = [torch.randn((p.n_halo, f), generator=g) for p in plans]            # every rank's halo-row gradient
    received = reverse_all_to_all(plans, halo_grads)
    ids = reverse_all_to_all(plans, [p.halo_ids for p in plans])
    for r, p in enumerate(plans):
        gp = check_reverse_plan(plans, r, ids[r])
        recv = torch.randn((received[r].size(0) + 2, ld), generator=g)              # padded pitch, 2 rows past the data
        recv[:received[r].size(0), :f] = received[r]
        before = recv.clone()
        grad = torch.randn((p.n_local + 3, ld), generator=g)                         # 3 rows past the rank's rows
        want = grad.clone()
        mask, send_off = (1 << gp.shift) - 1, _offsets(p.send_splits)
        for i in range(gp.n_rows):
            row = int(gp.rows[i])
            for v in gp.enc[int(gp.rowptr[i]):int(gp.rowptr[i + 1])].tolist():
                want[row, :f] = want[row, :f] + recv[send_off[v >> gp.shift] + (v & mask), :f]
        return_grad(emu, p, gp, recv, grad, f)
        assert torch.equal(grad, want), f"rank {r}"                                 # padding and other rows untouched too
        assert torch.equal(recv, before)                                             # the receive buffer is only read
    assert sum(p.n_halo for p in plans) > 0


@pytest.mark.parametrize("world,f,hub", [(2, 12, 600), (3, 8, 900), (4, 16, 0)])
def test_emulated_halo_backward_gives_the_whole_graph_gradient(emu, world, f, hub):
    n, e = 240, 2400
    src, dst, deg, bounds = partitioned_graph(n, e, world, seed=7 + world, hub=hub)
    plans = halo_plans(src, dst, bounds, world)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(n, f, generator=g)
    avg = O.avg_deg_from_histogram(torch.bincount(deg))
    w = torch.randn(n, len(A4) * len(S3) * f, generator=g)
    xr = x.clone().requires_grad_(True)
    (O.simple_propagate(xr, torch.stack([src, dst]), A4, S3, avg) * w).sum().backward()
    halo_grads, grads = [], []
    for p in plans:                                   # every rank: autograd on [local ; halo]
        ext = torch.cat([x[p.lo:p.hi], x[p.halo_ids]]).requires_grad_(True)
        out = O.simple_propagate(ext, torch.stack([p.src_ext, p.dst_local]), A4, S3, avg)[: p.n_local]
        (out * w[p.lo:p.hi]).sum().backward()
        halo_grads.append(ext.grad[p.n_local:].contiguous())
        grads.append(ext.grad[: p.n_local].clone())
    received = reverse_all_to_all(plans, halo_grads)
    for r, p in enumerate(plans):                     # every owner: add what came back
        return_grad(emu, p, pd.halo_grad_return_plan(p), received[r].contiguous(), grads[r], f)
    assert sum(p.n_halo for p in plans) > 0
    # the same per-edge terms, summed per rank and then across ranks: fp32 reordering only
    torch.testing.assert_close(torch.cat(grads), xr.grad, rtol=1e-5, atol=1e-5 * float(xr.grad.abs().max()))
