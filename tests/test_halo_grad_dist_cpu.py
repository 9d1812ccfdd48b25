"""The pull plane's reverse plan with real collectives on CPU: world_size-2 gloo processes build it with
``build_grad_return_plan`` (two all-to-alls) and it must be exactly what the pure builder makes from every rank's pull plan."""
import os
import socket
import sys

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


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
        from pna_b200 import dist as pd
        g = torch.Generator().manual_seed(11)
        n, e = 300, 3000
        src = torch.randint(0, n, (e,), generator=g)
        dst = torch.randint(0, int(n * 0.9), (e,), generator=g)
        dst[: e // 6] = 5
        bounds = pd.partition_bounds(torch.bincount(dst, minlength=n), world)
        plans = []
        for r in range(world):
            mine = (dst >= bounds[r]) & (dst < bounds[r + 1])
            plans.append(pd.build_pull_plan(src[mine], dst[mine], bounds, r, world))
        got = pd.build_grad_return_plan(plans[rank])
        want = pd.grad_return_plans(plans)[rank]
        assert got.shift == want.shift and got.peer_n_local == want.peer_n_local and (got.rank, got.world) == (rank, world)
        for name in ("rows", "rowptr", "enc"):
            a, b = getattr(got, name), getattr(want, name)
            assert a.dtype == b.dtype == torch.int32 and torch.equal(a, b), name
        q.put((rank, "ok", got.n_rows))
    except Exception:  # pragma: no cover
        import traceback
        q.put((rank, "fail: " + traceback.format_exc(), 0))
    finally:
        dist.destroy_process_group()


def test_distributed_reverse_plan_equals_the_pure_builder_world2():
    world, port = 2, _free_port()
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
    assert all(r[2] > 0 for r in res)                 # both ranks have rows held by the other
