"""The pull plane's backward on ONE GPU: W "ranks" in one process, every rank's feature and gradient buffers are ordinary
device tensors and the pointer tables name them all -- pna_halo_pull and pna_halo_grad_pull only see pointers, so the code
path is the one a multi-GPU run takes over NVLink.  The gradient that comes back to every owner must be the single-GPU
gradient of the whole graph, and the reference's autograd (CPU oracle)."""
import threading

import pytest
import torch

from oracle import pna_oracle as O

pytestmark = pytest.mark.gpu

A4 = ["mean", "max", "min", "std"]
A3 = ["mean", "std", "sum"]       # bf16 ties often; min/max routing of ties is checked in fp32 (tests/test_gpu_parity.py)
S3 = ["identity", "amplification", "attenuation"]


def dev():
    return torch.device("cuda:0")


def _graph(n, e, hub, seed):
    g = torch.Generator().manual_seed(seed)
    src = torch.randint(0, n, (e,), generator=g)
    dst = torch.randint(0, int(n * 0.93), (e,), generator=g)
    if hub:                                        # above the split threshold: the split-row backward
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.full((hub,), n // 3)])
        p = torch.randperm(src.numel(), generator=g)
        src, dst = src[p], dst[p]
    return src, dst


def _ranks(src, dst, n, f, world, dtype, barrier=None):
    """Pull plans, reverse plans and trainable aggregators of W ranks whose buffers are plain tensors on one GPU."""
    from pna_b200 import dist as pd
    deg = torch.bincount(dst, minlength=n)
    bounds = pd.partition_bounds(deg, world)
    plans = []
    for r in range(world):
        mine = (dst >= bounds[r]) & (dst < bounds[r + 1])
        plans.append(pd.build_pull_plan(src[mine].to(dev()), dst[mine].to(dev()), bounds, r, world))
    gplans = pd.grad_return_plans(plans)
    rows = max(p.n_local + p.n_halo for p in plans)
    feat = [[torch.zeros((rows, f), dtype=dtype, device=dev()) for _ in range(world)] for _ in range(2)]
    grad = [[torch.zeros((rows, f), dtype=torch.float32, device=dev()) for _ in range(world)] for _ in range(2)]
    flags = [torch.zeros(world, dtype=torch.int64, device=dev()) for _ in range(world)]

    def alloc_for(r):
        calls = {"i": 0}

        def alloc(shape, dt):      # call order: the feature buffers, the flags, the gradient buffers
            i = calls["i"]
            calls["i"] += 1
            pool = feat[i] if i < 2 else (flags if i == 2 else grad[i - 3])
            return pool[r], [t.data_ptr() for t in pool], None
        return alloc
    aggs = [pd.PullAggregator(plans[r], f, dtype=dtype, buffers=2, _alloc=alloc_for(r), trainable=True, grad_plan=gplans[r],
                              _barrier=barrier) for r in range(world)]
    return bounds, plans, aggs


def _oracle_grads(x, rb, src, dst, n, w, aggrs, avg, towers, with_self):
    """The reference's autograd: message x_j (+ row_bias_i), per tower [self block, aggregate]."""
    xr = x.float().clone().requires_grad_(True)
    br = None if rb is None else rb.float().clone().requires_grad_(True)
    msg = xr[src] + (br[dst] if br is not None else 0.0)
    ft = x.size(1) // towers
    blocks = []
    for t in range(towers):
        if with_self:
            blocks.append(xr[:, t * ft:(t + 1) * ft])
        blocks.append(O.pyg_aggregate(msg[:, t * ft:(t + 1) * ft], dst, n, aggrs, S3, avg))
    (torch.cat(blocks, 1) * w).sum().backward()
    return xr.grad, None if br is None else br.grad


@pytest.mark.parametrize("n,e,hub,f,world,dtype,towers,extras,mode", [
    (2000, 16000, 1500, 64, 2, torch.float32, 1, False, "atomic"),
    (1500, 10000, 0, 75, 3, torch.float32, 1, False, "coef"),
    (1800, 12000, 900, 128, 4, torch.float32, 2, True, "atomic"),
    (1200, 8000, 700, 256, 3, torch.float32, 4, True, "coef"),
    (1600, 11000, 800, 128, 4, torch.float32, 1, False, "coef"),
    (1200, 8000, 0, 64, 4, torch.bfloat16, 1, False, "atomic"),
    (1000, 7000, 500, 128, 2, torch.bfloat16, 2, True, "coef"),
])
def test_pull_plane_backward_phase_by_phase(n, e, hub, f, world, dtype, towers, extras, mode, monkeypatch):
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", mode)
    aggrs = A4 if dtype == torch.float32 else A3
    src, dst = _graph(n, e, hub, seed=n + f + world)
    g = torch.Generator().manual_seed(f)
    x = torch.randn(n, f, generator=g).to(dtype)
    rb = torch.randn(n, f, generator=g).to(dtype) if extras else None
    deg = torch.bincount(dst, minlength=n)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    width = towers * ((1 if extras else 0) + len(aggrs) * len(S3)) * (f // towers)
    w = torch.randn(n, width, generator=g)
    wd = w.to(dev())

    # the whole graph on one GPU
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    xg = x.to(dev()).requires_grad_(True)
    rbg = rb.to(dev()).requires_grad_(True) if extras else None
    out = pna_b200.pna_aggregate(xg, csr, aggrs, S3, avg, towers=towers, row_bias=rbg, self_feat=xg if extras else None)
    (out.float() * wd).sum().backward()

    # W ranks, phase by phase: forward everywhere, the aggregation's backward everywhere, stage everywhere, pull everywhere
    bounds, plans, aggs = _ranks(src, dst, n, f, world, dtype)
    xl = [x[int(bounds[r]):int(bounds[r + 1])].to(dev()) for r in range(world)]
    for r in range(world):                        # no barrier in one process: every rank's rows are written up front
        aggs[r].x_local.copy_(xl[r])
    exts, sfs, rbs = [], [], []
    for r in range(world):
        exts.append(aggs[r].exchange_features(xl[r]).requires_grad_(True))
        assert torch.equal(exts[r][plans[r].n_local:], x.to(dev())[plans[r].halo_ids])
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        sfs.append(xl[r].clone().requires_grad_(True) if extras else None)
        rbs.append(rb[lo:hi].to(dev()).requires_grad_(True) if extras else None)
        o = pna_b200.pna_aggregate(exts[r], aggs[r].csr, aggrs, S3, avg, towers=towers, row_bias=rbs[r], self_feat=sfs[r])
        assert torch.equal(o, out[lo:hi].detach())
        (o.float() * wd[lo:hi]).sum().backward()
    for r in range(world):
        aggs[r].stage_halo_grad(exts[r].grad)
    got = []
    for r in range(world):
        gr = aggs[r].pull_halo_grad(exts[r].grad)
        if extras:
            gr = gr + sfs[r].grad.float()
        got.append(gr)
    got = torch.cat(got).to(dtype).float().cpu()
    want = xg.grad.float().cpu()
    assert sum(p.n_halo for p in plans) > 0

    # same terms, other atomic order (and for bf16 the halo gradients are rounded before they are summed): vs. magnitude
    rel = 1e-4 if dtype == torch.float32 else 2e-2
    scale = float(want.abs().max())
    assert float((got - want).abs().max()) <= rel * scale, f"max diff {float((got - want).abs().max()):.3e} vs max |grad| {scale:.3e}"
    want_x, want_b = _oracle_grads(x, rb, src, dst, n, w, aggrs, avg, towers, extras)
    # bf16: x.grad is bf16 (2^-8 relative resolution) and is the sum of several bf16-rounded gradients that can be larger
    # than the result; the oracle runs in fp32 on the same inputs: a few bf16 steps of the largest entry
    tol = dict(rtol=1e-3, atol=5e-4) if dtype == torch.float32 else dict(rtol=5e-2, atol=2.0 ** -6 * float(want_x.abs().max()))
    torch.testing.assert_close(got, want_x, **tol)
    torch.testing.assert_close(want, want_x, **tol)
    if extras:
        gb = torch.cat([t.grad.float() for t in rbs]).cpu()
        torch.testing.assert_close(gb, rbg.grad.float().cpu(), rtol=0, atol=rel * float(rbg.grad.float().abs().max()))


@pytest.mark.parametrize("world,f,mode", [(2, 64, "atomic"), (3, 128, "coef"), (4, 64, "atomic")])
def test_pull_plane_trains_two_layers_like_one_gpu(world, f, mode, monkeypatch):
    """The autograd Function itself: one thread per rank, a host-side barrier (stream synchronize + threading.Barrier), two
    stacked layers through the same double-buffered aggregator, SGD on the all-reduced parameter gradients."""
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", mode)
    n, e, hub, steps, lr = 1500, 12000, 900, 3, 0.05
    src, dst = _graph(n, e, hub, seed=world * 7 + f)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(n, f, generator=g)
    deg = torch.bincount(dst, minlength=n)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    k = len(A4) * len(S3)
    # small weights keep tanh unsaturated: saturated neighbours (exactly +-1.0) give var = 0 rows, where the std slope (up to
    # 158) turns the backward's run-to-run atomic order into gradient noise far above what the exchange is checked to
    w1, w2 = 0.1 * torch.randn(k, f, generator=g) / k ** 0.5, 0.1 * torch.randn(k, f, generator=g) / k ** 0.5
    wout = torch.randn(n, f, generator=g)

    def mix(a, p):
        # row-wise weighted sum of the k aggregate blocks: elementwise ops only, so a rank's rows get the same bits as in
        # the whole-graph run (a GEMM may round differently for another row count) and the forwards stay identical
        a = a.view(a.size(0), k, f)
        acc = a[:, 0] * p[0]
        for j in range(1, k):
            acc = acc + a[:, j] * p[j]
        return acc

    def layers(agg_fn, xin, p):
        h = torch.tanh(mix(agg_fn(xin), p[0]))
        return mix(agg_fn(h), p[1])

    # one GPU
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    params = [w1.to(dev()).requires_grad_(True), w2.to(dev()).requires_grad_(True)]
    want = []
    for _ in range(steps):
        xg = x.to(dev()).requires_grad_(True)
        loss = (layers(lambda t: pna_b200.pna_aggregate(t, csr, A4, S3, avg), xg, params) * wout.to(dev())).sum()
        loss.backward()
        want.append((float(loss.detach()), xg.grad.cpu(), [p.grad.cpu() for p in params]))
        with torch.no_grad():
            for p in params:
                p -= lr * p.grad
                p.grad = None

    # W ranks, one thread each
    bar = threading.Barrier(world, timeout=120)

    def host_barrier():
        torch.cuda.current_stream().synchronize()
        bar.wait()
    bounds, plans, aggs = _ranks(src, dst, n, f, world, torch.float32, barrier=host_barrier)
    rparams = [[w1.to(dev()).requires_grad_(True), w2.to(dev()).requires_grad_(True)] for _ in range(world)]
    got = [[None] * world for _ in range(steps)]
    errors = []

    def rank_main(r):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        try:
            torch.cuda.set_device(0)
            # backward on this thread (not the shared device thread): its barrier waits for the other ranks' backward
            with torch.autograd.set_multithreading_enabled(False):
                for s in range(steps):
                    xr = x[lo:hi].to(dev()).requires_grad_(True)
                    out = layers(lambda t: aggs[r].pna_aggregate(t, A4, S3, avg), xr, rparams[r])
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
        except BaseException as exc:  # noqa: BLE001 -- reported below; the other ranks are released
            errors.append((r, exc))
            bar.abort()
    threads = [threading.Thread(target=rank_main, args=(r,)) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=600)
    assert not any(t.is_alive() for t in threads)
    assert not errors, errors
    for s in range(steps):
        loss_w, xgrad_w, pgrad_w = want[s]
        loss_g = sum(got[s][r][0] for r in range(world))
        assert abs(loss_g - loss_w) <= 1e-4 * max(1.0, abs(loss_w)), (s, loss_g, loss_w)
        xgrad_g = torch.cat([got[s][r][1] for r in range(world)])
        torch.testing.assert_close(xgrad_g, xgrad_w, rtol=1e-3, atol=5e-4 * max(1.0, float(xgrad_w.abs().max())))
        for a, b in zip(got[s][world], pgrad_w):
            assert float((a - b).norm() / b.norm().clamp(min=1e-6)) < 1e-3


def test_forward_only_aggregator_allocates_and_communicates_nothing_more(monkeypatch):
    from pna_b200 import dist as pd
    n, f, world = 600, 64, 2
    src, dst = _graph(n, 4000, 0, seed=3)
    deg = torch.bincount(dst, minlength=n)
    bounds = pd.partition_bounds(deg, world)
    plans = []
    for r in range(world):
        mine = (dst >= bounds[r]) & (dst < bounds[r + 1])
        plans.append(pd.build_pull_plan(src[mine].to(dev()), dst[mine].to(dev()), bounds, r, world))
    collectives = []
    for name in ("all_reduce", "all_to_all_single", "all_gather_object", "barrier", "all_gather"):
        monkeypatch.setattr(pd.dist, name, lambda *a, _n=name, **k: collectives.append(_n))
    shapes = []

    def alloc(shape, dt):
        shapes.append((tuple(shape), dt))
        t = torch.zeros(shape, dtype=dt, device=dev())
        return t, [t.data_ptr()] * world, None
    agg = pd.PullAggregator(plans[0], f, _alloc=alloc)
    assert len(shapes) == 3 and not collectives and agg.grad_plan is None    # two feature buffers and the flags
    x = torch.randn(plans[0].n_local, f, device=dev(), requires_grad=True)
    with pytest.raises(RuntimeError):
        agg.pna_aggregate(x, A4, S3, {"log": 1.0, "lin": 1.0})                 # a gradient needs trainable=True
    shapes.clear()
    agg = pd.PullAggregator(plans[0], f, _alloc=alloc, trainable=True, grad_plan=pd.grad_return_plans(plans)[0])
    assert len(shapes) == 5 and shapes[3][1] == torch.float32 and not collectives
