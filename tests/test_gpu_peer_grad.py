"""The peer plane's backward on ONE GPU: W "ranks" in one process, one thread each, whose ring slots, per-slot gradient
buffers and barrier flags are ordinary device tensors named by pointer tables -- pna_aggregate_fwd, pna_aggregate_bwd_peer_slots
and pna_halo_grad_pull only see pointers, so the code path is the one a multi-GPU run takes over NVLink; a host barrier
(stream synchronize + threading.Barrier) stands in for pna_peer_barrier.  The gradient every owner gets back must be the
single-GPU deterministic backward's bit for bit when no source has split_threshold out-slots or more, and a sequential fp32
sum of the whole graph's per-slot gradients when some do; the reference's fp32 autograd within the fp32 bar."""
import threading

import numpy as np
import pytest
import torch

from oracle import pna_oracle as O

pytestmark = pytest.mark.gpu

A6 = ["mean", "max", "min", "std", "sum", "var"]
A4 = ["mean", "std", "sum", "var"]        # bf16 ties often; min / max routing of ties is checked in fp32
S5 = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]


def dev():
    return torch.device("cuda:0")


def _graph(n, e, hub, hot, seed):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, int(n * 0.93), (e,), generator=g)       # the last rows have no in-edges
    if hub:                                                         # a destination above the split threshold
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.full((hub,), n // 3)])
    if hot:                                                         # a source with more out-slots than the split threshold
        src = torch.cat([src, torch.full((hot,), n // 2 + 1)])
        dst = torch.cat([dst, torch.randint(0, int(n * 0.93), (hot,), generator=g)])
    p = torch.randperm(src.numel(), generator=g)
    return src[p], dst[p]


def _ranks(src, dst, n, f, world, dtype, saved_layers=2, barrier=None):
    """Trainable peer aggregators of W ranks whose buffers are plain tensors on one GPU (allocated per call index, the same
    shape on every rank), with the reverse slot plans built in one process."""
    import pna_b200
    from pna_b200 import dist as pd
    deg = torch.bincount(dst, minlength=n)
    bounds = pd.partition_bounds(deg, world)
    shift = pd.peer_shift_for(bounds)
    cols = []
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        mine = (dst >= lo) & (dst < hi)
        enc = pd.encode_peer_sources(src[mine].to(dev()), bounds, shift)
        cols.append(pna_b200.build_csr(enc, dst[mine].to(dev()) - lo, hi - lo, n_src=world << shift).col)
    gplans = pd.peer_grad_return_plans(cols, shift)
    pools = {}

    def alloc_for(r):
        calls = {"i": 0}

        def alloc(shape, dt):
            i = calls["i"]
            calls["i"] += 1
            if i not in pools:
                pools[i] = [torch.zeros(shape, dtype=dt, device=dev()) for _ in range(world)]
            assert tuple(pools[i][r].shape) == tuple(shape) and pools[i][r].dtype == dt
            return pools[i][r], [t.data_ptr() for t in pools[i]], None
        return alloc
    aggs = []
    for r in range(world):
        mine = (dst >= bounds[r]) & (dst < bounds[r + 1])
        aggs.append(pd.PeerAggregator(src[mine].to(dev()), dst[mine].to(dev()), bounds, r, world, f, dtype=dtype, trainable=True,
                                      saved_layers=saved_layers, grad_plan=gplans[r], _alloc=alloc_for(r), _barrier=barrier))
    return bounds, aggs


def _run_ranks(world, fn):
    """fn(r, host_barrier) on one thread per rank; the backward runs on the rank's own thread."""
    bar = threading.Barrier(world, timeout=180)
    errors = []

    def host_barrier():
        torch.cuda.current_stream().synchronize()
        bar.wait()

    def main(r):
        try:
            torch.cuda.set_device(0)
            with torch.autograd.set_multithreading_enabled(False):
                fn(r, host_barrier)
        except BaseException as exc:  # noqa: BLE001 -- reported below; the other ranks are released
            errors.append((r, exc))
            bar.abort()
    threads = [threading.Thread(target=main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=900)
    assert not any(t.is_alive() for t in threads)
    assert not errors, errors
    return host_barrier


def _slot_grads(xg, rbg, w, csr, aggrs, avg, towers, has_self):
    """The whole graph's per-slot gradients (deterministic backward of the messages x[col] (+ row_bias) in CSR order)."""
    from pna_b200 import aggregate as ag
    msgs = xg.detach()[csr.col.long()]
    with torch.no_grad():
        torch.use_deterministic_algorithms(True)
        try:
            gs, _ = ag.aggregate_backward(w, msgs, csr, aggrs, S5, avg, towers=towers,
                                          row_bias=None if rbg is None else rbg.detach(), has_self=has_self,
                                          messages_in_csr_order=True)
        finally:
            torch.use_deterministic_algorithms(False)
    return gs


CASES = [   # n, e, hub, hot, f, world, dtype, towers, extras
    (2000, 16000, 900, 0, 64, 2, torch.float32, 1, True),
    (1500, 10000, 0, 0, 75, 3, torch.float32, 1, False),
    (1800, 12000, 700, 0, 128, 8, torch.float32, 2, True),
    (1200, 8000, 600, 0, 64, 3, torch.bfloat16, 1, True),
    (1600, 11000, 800, 1200, 128, 3, torch.float32, 1, True),
    (1000, 7000, 500, 900, 80, 2, torch.bfloat16, 2, True),
    (1400, 9000, 0, 700, 75, 8, torch.float32, 1, False),
]


@pytest.mark.parametrize("n,e,hub,hot,f,world,dtype,towers,extras", CASES)
def test_peer_plane_backward_equals_one_gpu(n, e, hub, hot, f, world, dtype, towers, extras, monkeypatch):
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", "coef")                       # ignored by the peer plane: always per-slot
    aggrs = A6 if dtype == torch.float32 else A4
    src, dst = _graph(n, e, hub, hot, seed=n + f + world)
    g = torch.Generator().manual_seed(f + world)
    x = torch.randn(n, f, generator=g).to(dtype)
    rb = torch.randn(n, f, generator=g).to(dtype) if extras else None
    sf = torch.randn(n, f, generator=g).to(dtype) if extras else None
    deg = torch.bincount(dst, minlength=n)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    width = towers * ((1 if extras else 0) + len(aggrs) * len(S5)) * (f // towers)
    w = torch.randn(n, width, generator=g).to(dtype)
    wd = w.to(dev())

    # the whole graph on one GPU, deterministic backward
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    xg = x.to(dev()).requires_grad_(True)
    rbg = rb.to(dev()).requires_grad_(True) if extras else None
    sfg = sf.to(dev()).requires_grad_(True) if extras else None
    out = pna_b200.pna_aggregate(xg, csr, aggrs, S5, avg, towers=towers, row_bias=rbg, self_feat=sfg)
    torch.use_deterministic_algorithms(True)
    try:
        out.backward(wd)
    finally:
        torch.use_deterministic_algorithms(False)

    bounds, aggs = _ranks(src, dst, n, f, world, dtype)
    res = [None] * world

    def rank(r, host_barrier):
        aggs[r]._barrier_hook = host_barrier
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        xr = x[lo:hi].to(dev()).requires_grad_(True)
        rbr = rb[lo:hi].to(dev()).requires_grad_(True) if extras else None
        sfr = sf[lo:hi].to(dev()).requires_grad_(True) if extras else None
        o = aggs[r].pna_aggregate(xr, aggrs, S5, avg, towers=towers, row_bias=rbr, self_feat=sfr)
        o.backward(wd[lo:hi])
        res[r] = (o.detach(), xr.grad, None if rbr is None else rbr.grad, None if sfr is None else sfr.grad)
    _run_ranks(world, rank)

    got_out = torch.cat([t[0] for t in res])
    assert torch.equal(got_out, out.detach())                          # the peer forward from the ring slot
    got = torch.cat([t[1] for t in res])
    hot_src = int(torch.bincount(src, minlength=n).max()) >= csr.split_threshold
    if not hot_src:
        assert torch.equal(got, xg.grad)                               # the single-GPU deterministic backward, bit for bit
    else:
        gs = _slot_grads(xg, rbg, wd, csr, aggrs, avg, towers, extras).cpu().numpy()
        want = np.zeros((n, f), dtype=np.float32)
        np.add.at(want, csr.col.long().cpu().numpy(), gs)            # each source's slots in ascending slot order, fp32
        assert torch.equal(got.float().cpu(), torch.from_numpy(want).to(dtype).float())
        torch.testing.assert_close(got.float(), xg.grad.float(), rtol=1e-3, atol=1e-3 * float(xg.grad.float().abs().max()))
    if extras:
        assert torch.equal(torch.cat([t[2] for t in res]), rbg.grad)
        assert torch.equal(torch.cat([t[3] for t in res]), sfg.grad)
    if dtype == torch.float32 and hot_src:
        # with hot sources the sum order is the peer plane's own: also the reference's autograd (fp32, as
        # tests/test_gpu_halo_grad.py checks the pull plane), at the same bar.  Without them the gradient is the single-GPU
        # one, bit for bit (above), whose agreement with the reference is tested on its own
        xo = x.clone().requires_grad_(True)
        bo = rb.clone().requires_grad_(True) if extras else None
        msg = xo[src] + (bo[dst] if extras else 0.0)
        ft = f // towers
        blocks = []
        for t in range(towers):
            if extras:
                blocks.append(sf[:, t * ft:(t + 1) * ft])
            blocks.append(O.pyg_aggregate(msg[:, t * ft:(t + 1) * ft], dst, n, aggrs, S5, avg))
        (torch.cat(blocks, 1) * w).sum().backward()
        torch.testing.assert_close(got.cpu(), xo.grad, rtol=1e-3, atol=5e-4 * max(1.0, float(xo.grad.abs().max())))


@pytest.mark.parametrize("world,f", [(2, 64), (3, 75), (8, 32)])
def test_peer_plane_trains_two_layers_like_one_gpu(world, f):
    """The autograd Function itself: one thread per rank, two stacked layers through one aggregator (saved_layers = 2),
    SGD on the all-reduced parameter gradients; x's gradient is the single-GPU deterministic one and two runs are
    bit-identical."""
    import pna_b200
    n, e, hub, steps, lr = 1500, 12000, 900, 3, 0.05
    src, dst = _graph(n, e, hub, 0, seed=world * 7 + f)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(n, f, generator=g)
    deg = torch.bincount(dst, minlength=n)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    aggrs = ["mean", "max", "min", "std"]
    scalers = S5[:3]
    k = len(aggrs) * len(scalers)
    w1, w2 = 0.1 * torch.randn(k, f, generator=g) / k ** 0.5, 0.1 * torch.randn(k, f, generator=g) / k ** 0.5
    wout = torch.randn(n, f, generator=g)

    def mix(a, p):
        # row-wise weighted sum of the k aggregate blocks: elementwise ops only, so a rank's rows get the same bits as in
        # the whole-graph run
        a = a.view(a.size(0), k, f)
        acc = a[:, 0] * p[0]
        for j in range(1, k):
            acc = acc + a[:, j] * p[j]
        return acc

    def layers(agg_fn, xin, p):
        h = torch.tanh(mix(agg_fn(xin), p[0]))
        return mix(agg_fn(h), p[1])

    # one GPU, deterministic backward
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    params = [w1.to(dev()).requires_grad_(True), w2.to(dev()).requires_grad_(True)]
    want = []
    torch.use_deterministic_algorithms(True)
    try:
        for _ in range(steps):
            xg = x.to(dev()).requires_grad_(True)
            loss = (layers(lambda t: pna_b200.pna_aggregate(t, csr, aggrs, scalers, avg), xg, params) * wout.to(dev())).sum()
            loss.backward()
            want.append((float(loss.detach()), xg.grad.cpu(), [p.grad.cpu() for p in params]))
            with torch.no_grad():
                for p in params:
                    p -= lr * p.grad
                    p.grad = None
    finally:
        torch.use_deterministic_algorithms(False)

    def run():
        bounds, aggs = _ranks(src, dst, n, f, world, torch.float32)
        rparams = [[w1.to(dev()).requires_grad_(True), w2.to(dev()).requires_grad_(True)] for _ in range(world)]
        got = [[None] * world for _ in range(steps)]

        def rank(r, host_barrier):
            aggs[r]._barrier_hook = host_barrier
            lo, hi = int(bounds[r]), int(bounds[r + 1])
            for s in range(steps):
                xr = x[lo:hi].to(dev()).requires_grad_(True)
                out = layers(lambda t: aggs[r].pna_aggregate(t, aggrs, scalers, avg), xr, rparams[r])
                loss = (out * wout[lo:hi].to(dev())).sum()
                loss.backward()
                got[s][r] = (float(loss.detach()), xr.grad.cpu())
                host_barrier()              # every rank's partial parameter gradients are complete: all-reduce them
                summed = [sum(rparams[q][i].grad for q in range(world)) for i in range(2)]
                host_barrier()
                with torch.no_grad():
                    for p, gsum in zip(rparams[r], summed):
                        p -= lr * gsum
                        p.grad = None
                if r == 0:
                    got[s].append([t.cpu() for t in summed])
        _run_ranks(world, rank)
        return got

    got, again = run(), run()
    for s in range(steps):
        loss_w, xgrad_w, pgrad_w = want[s]
        loss_g = sum(got[s][r][0] for r in range(world))
        assert abs(loss_g - loss_w) <= 1e-4 * max(1.0, abs(loss_w)), (s, loss_g, loss_w)
        xgrad_g = torch.cat([got[s][r][1] for r in range(world)])
        if s == 0:
            assert torch.equal(xgrad_g, xgrad_w)                       # same parameters: the same bits as one GPU
        torch.testing.assert_close(xgrad_g, xgrad_w, rtol=1e-3, atol=5e-4 * max(1.0, float(xgrad_w.abs().max())))
        for a, b in zip(got[s][world], pgrad_w):
            assert float((a - b).norm() / b.norm().clamp(min=1e-6)) < 1e-3
        for r in range(world):                                          # two runs: the same bits
            assert got[s][r][0] == again[s][r][0] and torch.equal(got[s][r][1], again[s][r][1])
        for a, b in zip(got[s][world], again[s][world]):
            assert torch.equal(a, b)


def test_forward_only_allocates_nothing_more_and_misuse_raises(monkeypatch):
    from pna_b200 import dist as pd
    n, f, world = 600, 64, 2
    src, dst = _graph(n, 4000, 0, 0, seed=3)
    deg = torch.bincount(dst, minlength=n)
    bounds = pd.partition_bounds(deg, world)
    mine = dst < bounds[1]
    collectives = []
    for name in ("all_reduce", "all_to_all_single", "all_gather_object", "barrier", "all_gather"):
        monkeypatch.setattr(pd.dist, name, lambda *a, _n=name, **k: collectives.append(_n))
    shapes = []

    def alloc(shape, dt):
        shapes.append((tuple(shape), dt))
        t = torch.zeros(shape, dtype=dt, device=dev())
        return t, [t.data_ptr()] * world, None
    s0, d0 = src[mine].to(dev()), dst[mine].to(dev())
    agg = pd.PeerAggregator(s0, d0, bounds, 0, world, f, _alloc=alloc)
    assert len(shapes) == 1 and not collectives and agg.grad_plan is None          # x_local only
    x = torch.randn(int(bounds[1]), f, device=dev(), requires_grad=True)
    avg = {"log": 1.0, "lin": 1.0}
    with pytest.raises(RuntimeError):
        agg.pna_aggregate(x, A6, S5, avg)                                           # needs trainable=True
    with pytest.raises(ValueError):
        pd.PeerAggregator(s0, d0, bounds, 0, world, f, _alloc=alloc, trainable=True, saved_layers=1, _barrier=lambda: None)
    # one rank's view of a 2-rank graph, barrier hook a no-op, its own ring slot standing in for the peer's
    cols = [pd.PeerAggregator(src[m].to(dev()), dst[m].to(dev()), bounds, r, world, f, _alloc=alloc).csr.col
            for r, m in enumerate([mine, ~mine])]
    gplan = pd.peer_grad_return_plans(cols, pd.peer_shift_for(bounds))[0]
    shapes.clear()
    agg = pd.PeerAggregator(s0, d0, bounds, 0, world, f, _alloc=alloc, trainable=True, saved_layers=2, grad_plan=gplan,
                            _barrier=lambda: None)
    assert len(shapes) == 1 + 2 + 1 + 2 and shapes[3][1] == torch.int64 and shapes[4][1] == torch.float32 and not collectives
    with pytest.raises(ValueError):
        pd.PeerAggregator(s0, d0, bounds, 0, world, f, _alloc=alloc, trainable=True,
                          grad_plan=pd.peer_grad_return_plans(cols, pd.peer_shift_for(bounds))[1], _barrier=lambda: None)
    with pytest.raises(ValueError):
        agg.pna_aggregate(x, ["mean", "softmax"], S5, avg)                        # the peer forward refuses them too
    outs = [agg.pna_aggregate(x, A6, S5, avg) for _ in range(2)]
    with pytest.raises(RuntimeError):
        agg.pna_aggregate(x, A6, S5, avg)                                           # a third call before any backward
    with torch.no_grad():
        agg.pna_aggregate(x, A6, S5, avg)                                           # no gradient: allowed, rewrites slot 0
    with pytest.raises(RuntimeError):
        outs[0].sum().backward()                                                    # its saved slot was rewritten
