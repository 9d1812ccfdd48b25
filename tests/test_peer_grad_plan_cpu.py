"""The peer plane's reverse slot plan on CPU: the pure builder (every rank in one process) names every slot of every rank
exactly once, at the owner of its source row, in ascending (rank, slot) order per row; world-size-2 and -3 gloo processes
build it with build_peer_grad_return_plan (two all-to-alls) and must get exactly the same plan."""
import os
import socket
import sys

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from pna_b200 import dist as pd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cols(n, e, world, seed):
    """Every rank's CSR col (owner << shift | row, destination-sorted, stable) of a random multigraph with a hot source."""
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, int(n * 0.9), (e,), generator=g)
    src[: e // 5] = 3                                                  # one source gathered by many slots on every rank
    bounds = pd.partition_bounds(torch.bincount(dst, minlength=n), world)
    shift = pd.peer_shift_for(bounds)
    cols = []
    for r in range(world):
        mine = (dst >= bounds[r]) & (dst < bounds[r + 1])
        order = torch.sort(dst[mine], stable=True).indices
        cols.append(pd.encode_peer_sources(src[mine][order], bounds, shift).to(torch.int32))
    return cols, shift, bounds


@pytest.mark.parametrize("world,n,e", [(1, 50, 300), (2, 300, 3000), (3, 400, 2500), (8, 500, 4000)])
def test_every_slot_once_in_ascending_rank_slot_order(world, n, e):
    cols, shift, bounds = _cols(n, e, world, seed=world)
    plans = pd.peer_grad_return_plans(cols, shift)
    seen = set()
    for r, gp in enumerate(plans):
        assert (gp.rank, gp.world) == (r, world) and gp.peer_n_edges == [c.numel() for c in cols]
        assert (world << gp.shift) < 2 ** 31 and max(c.numel() for c in cols) <= (1 << gp.shift)
        rows, rowptr, enc = gp.rows.long(), gp.rowptr.long(), gp.enc.long()
        assert gp.rows.dtype == gp.rowptr.dtype == gp.enc.dtype == torch.int32
        assert bool((rows[1:] > rows[:-1]).all()) and int(rowptr[0]) == 0 and int(rowptr[-1]) == enc.numel()
        for i in range(rows.numel()):
            ks = enc[rowptr[i]:rowptr[i + 1]].tolist()
            assert len(ks) >= 1 and ks == sorted(ks)                    # ascending (rank, slot): rank in the high bits
            for k in ks:
                p, s = k >> gp.shift, k & ((1 << gp.shift) - 1)
                c = int(cols[p][s])
                assert (c >> shift, c & ((1 << shift) - 1)) == (r, int(rows[i]))   # the slot gathers this row
                assert (p, s) not in seen
                seen.add((p, s))
    assert len(seen) == sum(c.numel() for c in cols)                   # every slot of every rank, exactly once


def test_shift_covers_the_largest_rank_and_refuses_overflow():
    gp = pd.peer_grad_return_plan(0, 2, [torch.zeros(0, dtype=torch.int64)] * 2, [torch.zeros(0, dtype=torch.int64)] * 2, [5, 1000])
    assert gp.shift == 10 and gp.n_rows == 0 and gp.rowptr.tolist() == [0]
    with pytest.raises(ValueError):
        pd.peer_grad_return_plan(0, 4, [torch.zeros(0, dtype=torch.int64)] * 4, [torch.zeros(0, dtype=torch.int64)] * 4,
                                 [1 << 29, 1, 1, 1])                     # 4 << 29 = 2^31


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from pna_b200 import dist as pdw
        cols, shift, _ = _cols(300, 3000, world, seed=20 + world)
        got = pdw.build_peer_grad_return_plan(cols[rank], shift, rank, world)
        want = pdw.peer_grad_return_plans(cols, shift)[rank]
        assert got.shift == want.shift and got.peer_n_edges == want.peer_n_edges and (got.rank, got.world) == (rank, world)
        for name in ("rows", "rowptr", "enc"):
            a, b = getattr(got, name), getattr(want, name)
            assert a.dtype == b.dtype == torch.int32 and torch.equal(a, b), name
        q.put((rank, "ok", got.n_rows))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), 0))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_distributed_reverse_slot_plan_equals_the_pure_builder(world):
    port = _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=180) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    for r in res:
        assert r[1] == "ok", r[1]
    assert all(r[2] > 0 for r in res)
