"""The halo plane's backward on ONE GPU: W "ranks" as threads of one process, the all-to-all replaced through
``HaloAggregator(_all_to_all=...)`` by copies between the ranks' device tensors (tests/test_halo_plane_grad_cpu.py's
ThreadedAllToAll); pack, aggregation and gradient return are the kernels a multi-GPU run calls.  Every rank's forward must
be the single-GPU rows bit for bit, its x.grad the single-GPU gradient of its rows and the oracle's; under
torch.use_deterministic_algorithms the gradients repeat bit for bit and equal the pull plane's."""
import threading

import pytest
import torch

from test_gpu_halo_grad import A3, A4, S3, _graph, _oracle_grads, _ranks as _pull_ranks
from test_halo_plane_grad_cpu import ThreadedAllToAll, halo_plans, run_ranks

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def _on_device(plan):
    from dataclasses import replace
    return replace(plan, **{k: getattr(plan, k).to(dev()) for k in ("src_ext", "dst_local", "halo_ids", "send_idx", "interior")})


def _halo_ranks(src, dst, n, f, world, dtype):
    """Halo plans and trainable aggregators of W in-process ranks sharing one ThreadedAllToAll (rank = group)."""
    from pna_b200 import dist as pd
    bounds = pd.partition_bounds(torch.bincount(dst, minlength=n), world)
    plans = [_on_device(p) for p in halo_plans(src, dst, bounds, world)]
    a2a = ThreadedAllToAll(world)
    aggs = [pd.HaloAggregator(plans[r], f, dtype=dtype, group=r, trainable=True, _all_to_all=a2a) for r in range(world)]
    return bounds, plans, aggs, a2a


def _on_threads(world, fn, abort):
    """fn(r) on one thread per rank; the backward runs on that thread (its all-to-all waits for the other ranks)."""
    def main(r):
        torch.cuda.set_device(0)
        with torch.autograd.set_multithreading_enabled(False):
            return fn(r)
    return run_ranks(world, main, abort=abort)


def _one_layer(aggregate, bounds, x, rb, wd, aggrs, avg, towers, extras):
    """Per rank: forward, (out * w).sum().backward(); returns (out, x.grad, row_bias.grad)."""
    def rank(r):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        xr = x[lo:hi].to(dev()).requires_grad_(True)
        rbr = rb[lo:hi].to(dev()).requires_grad_(True) if extras else None
        o = aggregate(r, xr, aggrs, S3, avg, towers=towers, row_bias=rbr, self_feat=xr if extras else None)
        (o.float() * wd[lo:hi]).sum().backward()
        return o.detach(), xr.grad, rbr.grad if extras else None
    return rank


@pytest.mark.parametrize("n,e,hub,f,world,dtype,towers,extras,mode", [
    (2000, 16000, 1500, 64, 2, torch.float32, 1, False, "atomic"),
    (1500, 10000, 0, 75, 3, torch.float32, 1, False, "coef"),
    (1800, 12000, 900, 128, 4, torch.float32, 2, True, "deterministic"),
    (1200, 8000, 700, 256, 3, torch.float32, 4, True, "atomic"),
    (1600, 11000, 800, 128, 4, torch.float32, 1, False, "coef"),
    (1200, 8000, 0, 64, 4, torch.bfloat16, 1, False, "deterministic"),
    (1000, 7000, 500, 128, 2, torch.bfloat16, 2, True, "atomic"),
    (1400, 9000, 600, 64, 3, torch.bfloat16, 1, True, "coef"),
])
def test_halo_plane_backward_matches_one_gpu(n, e, hub, f, world, dtype, towers, extras, mode, monkeypatch):
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", "coef" if mode == "coef" else "atomic")
    if mode == "deterministic":
        monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
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
    torch.use_deterministic_algorithms(mode == "deterministic")
    try:
        # the whole graph on one GPU
        csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
        xg = x.to(dev()).requires_grad_(True)
        rbg = rb.to(dev()).requires_grad_(True) if extras else None
        out = pna_b200.pna_aggregate(xg, csr, aggrs, S3, avg, towers=towers, row_bias=rbg, self_feat=xg if extras else None)
        (out.float() * wd).sum().backward()
        # W ranks
        bounds, plans, aggs, a2a = _halo_ranks(src, dst, n, f, world, dtype)
        res = _on_threads(world, _one_layer(lambda r, *a, **k: aggs[r].pna_aggregate(*a, **k), bounds, x, rb, wd, aggrs, avg,
                                            towers, extras), abort=[a2a.abort])
    finally:
        torch.use_deterministic_algorithms(False)
    assert sum(p.n_halo for p in plans) > 0 and a2a.calls == 2          # one exchange forward, one backward
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        assert torch.equal(res[r][0], out[lo:hi].detach()), f"rank {r} forward"
        assert res[r][1].dtype == dtype
    got = torch.cat([t[1] for t in res]).float().cpu()
    want = xg.grad.float().cpu()
    # same terms, other order of the adds (and for bf16 the halo gradients are rounded before they are summed)
    rel = 1e-4 if dtype == torch.float32 else 2e-2
    scale = float(want.abs().max())
    assert float((got - want).abs().max()) <= rel * scale, f"max diff {float((got - want).abs().max()):.3e} vs max |grad| {scale:.3e}"
    want_x, _ = _oracle_grads(x, rb, src, dst, n, w, aggrs, avg, towers, extras)     # self block included, as in x.grad
    tol = dict(rtol=1e-3, atol=5e-4) if dtype == torch.float32 else dict(rtol=5e-2, atol=2.0 ** -6 * float(want_x.abs().max()))
    torch.testing.assert_close(got, want_x, **tol)
    if extras:
        gb = torch.cat([t[2] for t in res]).float().cpu()
        torch.testing.assert_close(gb, rbg.grad.float().cpu(), rtol=0, atol=rel * float(rbg.grad.float().abs().max()))


@pytest.mark.parametrize("world,f,dtype,hub,extras", [(3, 128, torch.float32, 900, True), (4, 64, torch.bfloat16, 0, False),
                                                      (2, 75, torch.float32, 600, True)])
def test_deterministic_halo_plane_repeats_and_equals_the_pull_plane(deterministic, world, f, dtype, hub, extras):
    import pna_b200
    n, e = 1500, 10000
    aggrs = A4 if dtype == torch.float32 else A3
    src, dst = _graph(n, e, hub, seed=world * 13 + f)
    g = torch.Generator().manual_seed(world + f)
    x = torch.randn(n, f, generator=g).to(dtype)
    rb = torch.randn(n, f, generator=g).to(dtype) if extras else None
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    width = ((1 if extras else 0) + len(aggrs) * len(S3)) * f
    wd = torch.randn(n, width, generator=g).to(dev())

    def halo_run():
        bounds, plans, aggs, a2a = _halo_ranks(src, dst, n, f, world, dtype)
        return bounds, _on_threads(world, _one_layer(lambda r, *a, **k: aggs[r].pna_aggregate(*a, **k), bounds, x, rb, wd,
                                                     aggrs, avg, 1, extras), abort=[a2a.abort])
    bounds, first = halo_run()
    _, second = halo_run()
    # the pull plane on the same graph: a host-side barrier in place of the device flag barrier
    bar = threading.Barrier(world, timeout=120)

    def host_barrier():
        torch.cuda.current_stream().synchronize()
        bar.wait()
    pbounds, _, paggs = _pull_ranks(src, dst, n, f, world, dtype, barrier=host_barrier)
    assert torch.equal(pbounds, bounds)
    pull = _on_threads(world, _one_layer(lambda r, *a, **k: paggs[r].pna_aggregate(*a, **k), bounds, x, rb, wd, aggrs, avg, 1,
                                         extras), abort=[bar.abort])
    for r in range(world):
        for a, b, c in zip(first[r], second[r], pull[r]):
            if a is None:
                continue
            assert torch.equal(a, b), f"rank {r}: two runs differ"
            assert torch.equal(a, c), f"rank {r}: halo and pull planes differ"


@pytest.mark.parametrize("world,f,mode", [(2, 64, "atomic"), (3, 128, "coef"), (4, 64, "atomic")])
def test_halo_plane_trains_two_layers_like_one_gpu(world, f, mode, monkeypatch):
    """One thread per rank, two stacked layers through the same aggregator, SGD on the all-reduced parameter gradients."""
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", mode)
    n, e, hub, steps, lr = 1500, 12000, 900, 3, 0.05
    src, dst = _graph(n, e, hub, seed=world * 7 + f)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(n, f, generator=g)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    k = len(A4) * len(S3)
    # small weights keep tanh unsaturated (tests/test_gpu_halo_grad.py explains why)
    w1, w2 = 0.1 * torch.randn(k, f, generator=g) / k ** 0.5, 0.1 * torch.randn(k, f, generator=g) / k ** 0.5
    wout = torch.randn(n, f, generator=g)

    def mix(a, p):   # elementwise, so a rank's rows get the same bits as in the whole-graph run
        a = a.view(a.size(0), k, f)
        acc = a[:, 0] * p[0]
        for j in range(1, k):
            acc = acc + a[:, j] * p[j]
        return acc

    def layers(agg_fn, xin, p):
        return mix(agg_fn(torch.tanh(mix(agg_fn(xin), p[0]))), p[1])

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

    bounds, plans, aggs, a2a = _halo_ranks(src, dst, n, f, world, torch.float32)
    rparams = [[w1.to(dev()).requires_grad_(True), w2.to(dev()).requires_grad_(True)] for _ in range(world)]
    bar = threading.Barrier(world, timeout=120)

    def host_barrier():
        torch.cuda.current_stream().synchronize()
        bar.wait()

    def rank(r):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        got = []
        for _ in range(steps):
            xr = x[lo:hi].to(dev()).requires_grad_(True)
            loss = (layers(lambda t: aggs[r].pna_aggregate(t, A4, S3, avg), xr, rparams[r]) * wout[lo:hi].to(dev())).sum()
            loss.backward()
            host_barrier()                  # every rank's partial parameter gradients are complete: all-reduce them
            summed = [sum(rparams[q][i].grad for q in range(world)) for i in range(2)]
            host_barrier()
            got.append((float(loss.detach()), xr.grad.cpu(), [t.cpu() for t in summed]))
            with torch.no_grad():
                for p, gsum in zip(rparams[r], summed):
                    p -= lr * gsum
                    p.grad = None
        return got
    res = _on_threads(world, rank, abort=[a2a.abort, bar.abort])
    assert a2a.calls == 4 * steps                       # two layers, one exchange each way
    for s in range(steps):
        loss_w, xgrad_w, pgrad_w = want[s]
        loss_g = sum(res[r][s][0] for r in range(world))
        assert abs(loss_g - loss_w) <= 1e-4 * max(1.0, abs(loss_w)), (s, loss_g, loss_w)
        xgrad_g = torch.cat([res[r][s][1] for r in range(world)])
        torch.testing.assert_close(xgrad_g, xgrad_w, rtol=1e-3, atol=5e-4 * max(1.0, float(xgrad_w.abs().max())))
        for a, b in zip(res[0][s][2], pgrad_w):
            assert float((a - b).norm() / b.norm().clamp(min=1e-6)) < 1e-3


def test_forward_only_halo_aggregator_allocates_and_communicates_nothing_more():
    import pna_b200
    from pna_b200 import dist as pd
    n, f, world = 600, 64, 2
    src, dst = _graph(n, 4000, 0, seed=3)
    bounds = pd.partition_bounds(torch.bincount(dst, minlength=n), world)
    plan = _on_device(halo_plans(src, dst, bounds, world)[0])
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    calls = []

    def a2a(output, input, output_split_sizes=None, input_split_sizes=None, group=None, async_op=False):
        calls.append((output.dtype, tuple(output.shape), list(output_split_sizes), list(input_split_sizes)))
        output.zero_()
    for overlap in (True, False):
        calls.clear()
        agg = pd.HaloAggregator(plan, f, overlap=overlap, _all_to_all=a2a)
        assert agg.grad_plan is None and agg._grad_recv is None and agg._grad_table is None and not calls
        agg.x_local.normal_()
        agg.aggregate(A4, S3, avg)
        assert calls == [(torch.float32, (plan.n_halo, f), plan.recv_splits, plan.send_splits)]
        x = torch.randn(plan.n_local, f, device=dev(), requires_grad=True)
        with pytest.raises(RuntimeError, match="trainable=True"):
            agg.pna_aggregate(x, A4, S3, avg)                               # a gradient needs trainable=True
        with pytest.raises(RuntimeError, match="trainable=True"):
            agg.return_halo_grad(torch.zeros(plan.n_local + plan.n_halo, f, device=dev()))
        assert len(calls) == 1
        with torch.no_grad():
            agg.pna_aggregate(x, A4, S3, avg)                               # forward only: allowed, one exchange
        assert len(calls) == 2
    calls.clear()
    agg = pd.HaloAggregator(plan, f, trainable=True, _all_to_all=a2a)
    assert not calls and agg.grad_plan.n_rows > 0 and agg.grad_plan.peer_n_local is None
    assert agg._grad_recv.dtype == torch.float32 and tuple(agg._grad_recv.shape) == (sum(plan.send_splits), f)
    mine = (dst >= bounds[0]) & (dst < bounds[1])
    pplan = pd.build_pull_plan(src[mine].to(dev()), dst[mine].to(dev()), bounds, 0, world)
    with pytest.raises(ValueError, match="peer_n_local"):                   # a pull plane cannot use the halo plane's plan
        pd.PullAggregator(pplan, f, _alloc=lambda shape, dt: (torch.zeros(shape, dtype=dt, device=dev()), [0] * world, None),
                          trainable=True, grad_plan=agg.grad_plan)
