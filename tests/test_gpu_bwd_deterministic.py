"""The deterministic backward on the GPU: under torch.use_deterministic_algorithms(True) the backward of pna_aggregate stores
per-slot gradients (pna_aggregate_bwd_slots) and sums them over the slot-transposed CSR with the forward kernel.  Two runs
must give the same bits; the result must match the reference's autograd (CPU oracle) and the atomic path to the
tolerances of tests/test_gpu_parity.py; the per-slot values must be the per-edge values of the atomic kernels, and the sums
of light source rows the sequential sums of those values in slot order."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

A4 = ["mean", "max", "min", "std"]
A3 = ["mean", "std", "sum"]              # bf16 ties often: min / max routing of ties is checked in fp32
AGGRS = ["sum", "mean", "min", "max", "var", "std"]
S3 = ["identity", "amplification", "attenuation"]
S5 = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]


def dev():
    return torch.device("cuda:0")


@pytest.fixture(scope="module", autouse=True)
def _release_memory():
    """These tests allocate up to ~1 GB of scratch; hand the cached blocks back so later modules start from a similar
    allocator state."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture
def deterministic(monkeypatch):
    """torch's switch on (PyTorch wants a fixed cuBLAS workspace under it); a spy counts the deterministic backward calls."""
    import pna_b200.aggregate as agg
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    calls = []
    real = agg._backward_deterministic

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(agg, "_backward_deterministic", spy)
    torch.use_deterministic_algorithms(True)
    try:
        yield calls
    finally:
        torch.use_deterministic_algorithms(False)


def rand_graph(n, e, seed, hub=0, hot_src=0, isolated=0.15):
    """Random multigraph; `hub` extra in-edges of the last row (split row), `hot_src` extra out-edges of row 0 (a split row of
    the reversed graph) -- or a Zipf-distributed source choice when hot_src < 0."""
    g = torch.Generator().manual_seed(seed)
    live = max(1, int(n * (1 - isolated)))
    dst = torch.randint(0, live, (e,), generator=g)
    if hot_src < 0:
        ranks = torch.arange(1, n + 1, dtype=torch.float64)
        src = torch.multinomial(1.0 / ranks, e, replacement=True, generator=g)
    else:
        src = torch.randint(0, n, (e,), generator=g)
    if hub:
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)]); dst = torch.cat([dst, torch.full((hub,), n - 1)])
    if hot_src > 0:
        src = torch.cat([src, torch.zeros(hot_src, dtype=torch.long)]); dst = torch.cat([dst, torch.randint(0, live, (hot_src,), generator=g)])
    p = torch.randperm(src.numel(), generator=g)
    return torch.stack([src[p], dst[p]])


def _avg(ei, n):
    from oracle import pna_oracle as O
    return O.avg_deg_from_histogram(torch.bincount(torch.bincount(ei[1], minlength=n)))


def _oracle(x, rb, ei, n, w, aggrs, scalers, avg, towers, with_self):
    from oracle import pna_oracle as O
    xr = x.float().clone().requires_grad_(True)
    br = None if rb is None else rb.float().clone().requires_grad_(True)
    src, dst = ei[0], ei[1]
    msg = xr[src] + (br[dst] if br is not None else 0.0)
    ft = x.size(1) // towers
    blocks = []
    for t in range(towers):
        if with_self:
            blocks.append(xr[:, t * ft:(t + 1) * ft])
        blocks.append(O.pyg_aggregate(msg[:, t * ft:(t + 1) * ft], dst, n, aggrs, scalers, avg))
    (torch.cat(blocks, 1) * w).sum().backward()
    return xr.grad, None if br is None else br.grad


def _run(csr, x, rb, w, aggrs, scalers, avg, towers, with_self):
    """One forward + backward through pna_aggregate; (grad x via gathered + self_feat, grad row_bias, grad self_feat)."""
    import pna_b200
    xg = x.to(dev()).requires_grad_(True)
    sf = x.to(dev()).requires_grad_(True) if with_self else None
    rbg = rb.to(dev()).requires_grad_(True) if rb is not None else None
    out = pna_b200.pna_aggregate(xg, csr, aggrs, scalers, avg, towers=towers, row_bias=rbg, self_feat=sf)
    (out.float() * w.to(dev())).sum().backward()
    return xg.grad, None if rb is None else rbg.grad, None if sf is None else sf.grad


CASES = [   # n, e, hub, hot_src, f, dtype, towers, extras
    (2000, 16000, 1500, 0, 64, torch.float32, 1, False),
    (1500, 12000, 900, 1200, 128, torch.float32, 2, True),       # split rows in both directions
    (3000, 30000, 0, -1, 96, torch.float32, 1, True),            # Zipf sources: the reversed graph has split rows
    (1200, 9000, 800, 0, 75, torch.float32, 3, True),            # scalar path (75 columns)
    (1500, 10000, 700, 900, 64, torch.bfloat16, 1, True),
    (1000, 7000, 0, -1, 128, torch.bfloat16, 2, False),
]


@pytest.mark.parametrize("n,e,hub,hot_src,f,dtype,towers,extras", CASES)
def test_backward_repeats_bit_for_bit_and_matches_the_oracle_and_the_atomic_path(deterministic, n, e, hub, hot_src, f, dtype, towers,
                                                                                 extras, monkeypatch):
    import pna_b200
    aggrs = A4 if dtype == torch.float32 else A3
    ei = rand_graph(n, e, seed=n + f, hub=hub, hot_src=hot_src)
    csr = pna_b200.build_csr(ei[0].to(dev()), ei[1].to(dev()), n)
    if hub:
        assert csr.n_hubs > 0
    if hot_src:
        assert csr.slot_transposed(n).n_hubs > 0
    g = torch.Generator().manual_seed(f)
    x = torch.randn(n, f, generator=g).to(dtype)
    rb = torch.randn(n, f, generator=g).to(dtype) if extras else None
    avg = _avg(ei, n)
    w = torch.randn(n, towers * ((1 if extras else 0) + len(aggrs) * len(S3)) * (f // towers), generator=g)
    first = _run(csr, x, rb, w, aggrs, S3, avg, towers, extras)
    second = _run(csr, x, rb, w, aggrs, S3, avg, towers, extras)
    assert len(deterministic) == 2
    for a, b in zip(first, second):
        assert (a is None) == (b is None)
        if a is not None:
            assert torch.equal(a, b)
    gx = first[0].float() + (first[2].float() if extras else 0.0)
    # the oracle and the atomic path: the bars of tests/test_gpu_parity.py / tests/test_gpu_halo_grad.py
    want_x, want_b = _oracle(x, rb, ei, n, w, aggrs, S3, avg, towers, extras)
    tol = dict(rtol=1e-3, atol=5e-4) if dtype == torch.float32 else dict(rtol=5e-2, atol=2.0 ** -6 * float(want_x.abs().max()))
    torch.testing.assert_close(gx.cpu(), want_x, **tol)
    torch.use_deterministic_algorithms(False)
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    atomic = _run(csr, x, rb, w, aggrs, S3, avg, towers, extras)
    torch.use_deterministic_algorithms(True)
    assert len(deterministic) == 2
    ga = atomic[0].float() + (atomic[2].float() if extras else 0.0)
    rel = 1e-4 if dtype == torch.float32 else 2e-2
    assert float((gx - ga).abs().max()) <= rel * float(ga.abs().max())
    if extras:
        # bf16: grad_out is rounded to bf16 before the backward, the oracle's is not; a split row sums 700 such terms
        tol_b = dict(rtol=1e-3, atol=2e-3) if dtype == torch.float32 else dict(rtol=5e-2, atol=2.0 ** -6 * float(want_b.abs().max()))
        torch.testing.assert_close(first[1].float().cpu(), want_b.float(), **tol_b)
        assert float((first[1].float() - atomic[1].float()).abs().max()) <= rel * float(atomic[1].float().abs().max())


def _descriptor(x, csr, aggrs, scalers, avg, towers, rb, in_order, scratch):
    from pna_b200 import _lib
    na, ac = _lib.pack_codes(aggrs, _lib.AGGR_CODES, "aggregator")
    ns, sc = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
    n, f = csr.n_nodes, x.size(1)
    return _lib.AggStruct(
        gathered=x.data_ptr(), ld_gathered=x.stride(0), rowptr=csr.rowptr.data_ptr(), col=None if in_order else csr.col.data_ptr(),
        row_bias=None if rb is None else rb.data_ptr(), ld_row_bias=0 if rb is None else rb.stride(0),
        n_rows=n, n_feat=f, n_towers=towers, dtype=_lib.PNA_F32 if x.dtype == torch.float32 else _lib.PNA_BF16,
        n_aggr=na, aggr_codes=ac, n_scalers=ns, scaler_codes=sc, avg_log=float(avg["log"]), avg_lin=float(avg["lin"]),
        split_threshold=csr.split_threshold, chunk_edges=csr.chunk_edges,
        hub_info=csr.hub_info.data_ptr() if csr.n_hubs else None, chunk_items=csr.chunk_items.data_ptr() if csr.n_hubs else None,
        n_hubs=csr.n_hubs, n_chunks=csr.n_chunks, hub_partials=None if scratch is None else scratch.data_ptr())


@pytest.mark.parametrize("f,dtype,with_bias", [(64, torch.float32, True), (75, torch.float32, False), (128, torch.bfloat16, True)])
def test_slots_are_the_per_slot_gradient_and_light_sources_the_ordered_sums(f, dtype, with_bias):
    """pna_aggregate_bwd_slots (through col) == pna_aggregate_bwd with col == NULL on the materialised messages x[col], bit for
    bit; and for sources below the split threshold the deterministic grad_gathered is the host's sequential fp32 sum of
    their slots' values in ascending slot order."""
    import pna_b200
    from pna_b200 import _lib
    n, e = 2000, 16000
    ei = rand_graph(n, e, seed=f, hub=1500, hot_src=1000)
    csr = pna_b200.build_csr(ei[0].to(dev()), ei[1].to(dev()), n)
    g = torch.Generator().manual_seed(7)
    x = torch.randn(n, f, generator=g).to(dtype).to(dev())
    rb = torch.randn(n, f, generator=g).to(dtype).to(dev()) if with_bias else None
    avg = _avg(ei, n)
    go = torch.randn(n, len(AGGRS) * len(S5) * f, generator=g).to(dtype).to(dev())
    scratch = torch.empty(((csr.n_chunks + csr.n_hubs) * 6, f), dtype=torch.float32, device=dev())
    E, L = csr.n_edges, _lib.lib()
    st = torch.cuda.current_stream().cuda_stream
    gs = torch.empty((E, f), dtype=torch.float32, device=dev())
    gb = torch.empty((n, f), dtype=torch.float32, device=dev()) if with_bias else None
    d = _descriptor(x, csr, AGGRS, S5, avg, 1, rb, False, scratch)
    _lib.check(L.pna_aggregate_bwd_slots(C.byref(d), go.data_ptr(), go.stride(0), 0, f, gs.data_ptr(), f,
                                         None if gb is None else gb.data_ptr(), f, st))
    xm = x[csr.col.long()].contiguous()
    want = torch.zeros((E, f), dtype=torch.float32, device=dev())
    gb2 = torch.empty((n, f), dtype=torch.float32, device=dev()) if with_bias else None
    d2 = _descriptor(xm, csr, AGGRS, S5, avg, 1, rb, True, scratch)
    _lib.check(L.pna_aggregate_bwd(C.byref(d2), go.data_ptr(), go.stride(0), want.data_ptr(), f, None if gb2 is None else gb2.data_ptr(),
                                   f, st))
    assert torch.equal(gs, want)
    # step 2 through the library's Python path, against the host's ordered sums for the light sources
    torch.use_deterministic_algorithms(True)
    try:
        gg, _ = pna_b200.aggregate.aggregate_backward(go, x, csr, AGGRS, S5, avg, row_bias=rb)
    finally:
        torch.use_deterministic_algorithms(False)
    col = csr.col.cpu().numpy()
    g_np = gs.cpu().numpy()
    acc = np.zeros((n, f), dtype=np.float32)
    for s in range(E):
        acc[col[s]] = acc[col[s]] + g_np[s]
    out_deg = np.bincount(col, minlength=n)
    light = out_deg < csr.split_threshold
    assert (~light).any() and light.sum() > n // 2
    assert np.array_equal(gg.cpu().numpy()[light], acc[light])
    np.testing.assert_allclose(gg.cpu().numpy()[~light], acc[~light], rtol=1e-4, atol=1e-4)


def test_slabs_equal_the_full_width_result(deterministic, monkeypatch):
    """DETERMINISTIC_SCRATCH_BYTES made small: the backward runs in feature slabs and must return the same bits."""
    import pna_b200
    import pna_b200.aggregate as agg
    n, e, f = 1500, 12000, 96
    ei = rand_graph(n, e, seed=5, hub=900, hot_src=700)
    csr = pna_b200.build_csr(ei[0].to(dev()), ei[1].to(dev()), n)
    g = torch.Generator().manual_seed(2)
    for dtype in (torch.float32, torch.bfloat16):
        x = torch.randn(n, f, generator=g).to(dtype)
        rb = torch.randn(n, f, generator=g).to(dtype)
        avg = _avg(ei, n)
        w = torch.randn(n, 2 * (1 + len(A3) * len(S3)) * (f // 2), generator=g)
        full = _run(csr, x, rb, w, A3, S3, avg, 2, True)
        for cols in (8, 24, 40):
            monkeypatch.setattr(agg, "DETERMINISTIC_SCRATCH_BYTES", csr.n_edges * 4 * cols)
            assert agg.deterministic_slab_width(csr.n_edges, f, 16 // x.element_size()) < f
            slabbed = _run(csr, x, rb, w, A3, S3, avg, 2, True)
            for a, b in zip(full, slabbed):
                assert torch.equal(a, b), (dtype, cols)
        monkeypatch.setattr(agg, "DETERMINISTIC_SCRATCH_BYTES", 1 << 30)


# ---- the layers reach the deterministic path through pna_aggregate ----------------------------------------------------
def _twice(fn):
    a, b = fn(), fn()
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    return a


def test_pyg_simple_conv(deterministic):
    import pna_b200 as P
    from oracle import pna_oracle as O
    n, e, f = 300, 2400, 16
    ei = rand_graph(n, e, seed=31, hub=400)
    x = torch.randn(n, f)
    deg = torch.bincount(torch.bincount(ei[1], minlength=n))
    ref = O.PNAConvSimpleOracle(f, f, A4, S3, deg)
    mine = P.PNAConvSimple(f, f, A4, S3, deg)
    mine.load_state_dict(ref.state_dict())
    mine = mine.to(dev())
    w = torch.randn(n, f)
    xr = x.clone().requires_grad_(True)
    (ref(xr, ei) * w).sum().backward()

    def run():
        mine.zero_grad()
        xm = x.clone().to(dev()).requires_grad_(True)
        (mine(xm, ei.to(dev())) * w.to(dev())).sum().backward()
        return xm.grad.clone(), mine.post_nn[0].weight.grad.clone()
    gx, gw = _twice(run)
    assert len(deterministic) == 2
    torch.testing.assert_close(gx.cpu(), xr.grad, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(gw.cpu(), ref.post_nn[0].weight.grad, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("name", ["pyg_conv_t1", "pyg_conv_t4_div", "pyg_conv_edge"])
def test_pyg_conv_affine_and_materialised_messages(deterministic, name):
    import pna_b200 as P
    from oracle import pna_oracle as O
    g = load_golden(name)
    c = g["ctor"]
    kw = dict(edge_dim=c["edge_dim"], towers=c["towers"], pre_layers=c["pre_layers"], post_layers=c["post_layers"],
              divide_input=c["divide_input"])
    ref = O.PNAConvOracle(c["in_channels"], c["out_channels"], g["aggregators"], g["scalers"], g["deg"], **kw)
    ref.load_state_dict(g["state_dict"])
    mine = P.PNAConv(c["in_channels"], c["out_channels"], g["aggregators"], g["scalers"], g["deg"], **kw)
    mine.load_state_dict(g["state_dict"])
    mine = mine.to(dev())
    x, ei, ea = g["x"], g["edge_index"], g["edge_attr"]
    w = torch.randn(x.size(0), c["out_channels"], generator=torch.Generator().manual_seed(0))
    xr = x.clone().requires_grad_(True)
    (ref(xr, ei, ea) * w).sum().backward()

    def run():
        mine.zero_grad()
        xm = x.clone().to(dev()).requires_grad_(True)
        (mine(xm, ei.to(dev()), None if ea is None else ea.to(dev())) * w.to(dev())).sum().backward()
        return [xm.grad.clone()] + [p.grad.clone() for _, p in sorted(mine.named_parameters())]
    got = _twice(run)
    assert len(deterministic) == 2
    torch.testing.assert_close(got[0].cpu(), xr.grad, rtol=1e-3, atol=5e-4)
    for gp, (n2, p2) in zip(got[1:], sorted(ref.named_parameters())):
        err = float((gp.cpu() - p2.grad).norm() / p2.grad.norm().clamp(min=1e-6))
        assert err < 2e-3, f"{n2}: relative Frobenius error {err:.2e}"


@pytest.mark.parametrize("name", ["dgl_layer_t5", "dgl_layer_edge", "dgl_simple", "dgl_simple_var"])
def test_dgl_layers(deterministic, monkeypatch, name):
    """DGL-signature layers (affine and per-edge messages, relu_var): repeat bit for bit; against the atomic backward at the
    bar the parity tests hold the atomic backward to the oracle."""
    import pna_b200 as P
    g = load_golden(name)
    simple = name.startswith("dgl_simple")
    cls = P.PNASimpleLayer if simple else P.PNALayer
    lay = cls(aggregators=g["aggregators"], scalers=g["scalers"], avg_d=g["avg_d"], **g["ctor"])
    lay.load_state_dict(g["state_dict"])
    lay = lay.to(dev()).eval()
    ei = g["edge_index"]
    gr = P.Graph(ei[0], ei[1], g["h"].size(0)).to(dev())
    e = None if simple or g["e"] is None else g["e"].to(dev())

    def run():
        lay.zero_grad()
        h = g["h"].clone().to(dev()).requires_grad_(True)
        out = lay(gr, h) if simple else lay(gr, h, e, g["snorm_n"].to(dev()))
        w = torch.randn(out.shape, generator=torch.Generator().manual_seed(1)).to(dev())
        (out * w).sum().backward()
        return [h.grad.clone()] + [p.grad.clone() for _, p in sorted(lay.named_parameters()) if p.grad is not None]
    got = _twice(run)
    assert len(deterministic) == 2
    torch.use_deterministic_algorithms(False)
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    want = run()
    torch.use_deterministic_algorithms(True)
    torch.testing.assert_close(got[0], want[0], rtol=1e-3, atol=5e-4)
    for a, b in zip(got[1:], want[1:]):
        assert float((a - b).norm() / b.norm().clamp(min=1e-6)) < 2e-3


def test_dense_layer_with_scaler_degree(deterministic):
    import pna_b200 as P
    g = load_golden("dense_k1_k2")
    lay = P.dense.PNALayer(aggregators=A4, scalers=S3, avg_d=g["avg_d"], **g["ctor"])
    lay.load_state_dict(g["state_dict"])
    lay = lay.to(dev()).eval()

    def run():
        lay.zero_grad()
        h = g["h"].clone().to(dev()).requires_grad_(True)
        (lay(h, g["adj"].to(dev())) * g["grads"]["w"].to(dev())).sum().backward()
        return [h.grad.clone()] + [p.grad.clone() for _, p in lay.named_parameters()]
    got = _twice(run)
    assert len(deterministic) >= 2
    torch.testing.assert_close(got[0].cpu(), g["grads"]["h"], rtol=1e-3, atol=5e-4)
    for (k, _), gp in zip(lay.named_parameters(), got[1:]):
        ref = g["grads"]["params"][k]
        assert float((gp.cpu() - ref).norm() / ref.norm().clamp(min=1e-6)) < 2e-3, k


# ---- the pull plane: W ranks in one process (the harness of tests/test_gpu_halo_grad.py) ------------------------------
def _train_ranks(src, dst, n, f, world, x, w1, w2, wout, avg, steps=2, lr=0.05):
    import threading
    from test_gpu_halo_grad import A4 as HA4, S3 as HS3, _ranks
    k = len(HA4) * len(HS3)

    def mix(a, p):
        a = a.view(a.size(0), k, f)
        acc = a[:, 0] * p[0]
        for j in range(1, k):
            acc = acc + a[:, j] * p[j]
        return acc

    def layers(agg_fn, xin, p):
        return mix(agg_fn(torch.tanh(mix(agg_fn(xin), p[0]))), p[1])

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
            with torch.autograd.set_multithreading_enabled(False):
                for s in range(steps):
                    xr = x[lo:hi].to(dev()).requires_grad_(True)
                    loss = (layers(lambda t: aggs[r].pna_aggregate(t, HA4, HS3, avg), xr, rparams[r]) * wout[lo:hi].to(dev())).sum()
                    loss.backward()
                    got[s][r] = (xr.grad.cpu(), [p.grad.cpu() for p in rparams[r]])
                    host_barrier()
                    summed = [sum(rparams[q][i].grad for q in range(world)) for i in range(2)]
                    host_barrier()
                    with torch.no_grad():
                        for p, gsum in zip(rparams[r], summed):
                            p -= lr * gsum
                            p.grad = None
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
    return got, layers


@pytest.mark.parametrize("world,f", [(2, 64), (3, 128)])
def test_pull_plane_training_repeats_bit_for_bit(deterministic, world, f):
    import pna_b200
    from test_gpu_halo_grad import A4 as HA4, S3 as HS3, _graph
    n, e, hub = 1500, 12000, 900
    src, dst = _graph(n, e, hub, seed=world * 11 + f)
    g = torch.Generator().manual_seed(world)
    x = torch.randn(n, f, generator=g)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    k = len(HA4) * len(HS3)
    w1, w2 = 0.1 * torch.randn(k, f, generator=g) / k ** 0.5, 0.1 * torch.randn(k, f, generator=g) / k ** 0.5
    wout = torch.randn(n, f, generator=g)
    run1, layers = _train_ranks(src, dst, n, f, world, x, w1, w2, wout, avg)
    run2, _ = _train_ranks(src, dst, n, f, world, x, w1, w2, wout, avg)
    assert len(deterministic) > 0
    for s1, s2 in zip(run1, run2):
        for (gx1, gp1), (gx2, gp2) in zip(s1, s2):
            assert torch.equal(gx1, gx2)
            for a, b in zip(gp1, gp2):
                assert torch.equal(a, b)
    # first step against the whole graph on one GPU
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    params = [w1.to(dev()).requires_grad_(True), w2.to(dev()).requires_grad_(True)]
    xg = x.to(dev()).requires_grad_(True)
    (layers(lambda t: pna_b200.pna_aggregate(t, csr, HA4, HS3, avg), xg, params) * wout.to(dev())).sum().backward()
    want = xg.grad.cpu()
    got = torch.cat([run1[0][r][0] for r in range(world)])
    torch.testing.assert_close(got, want, rtol=1e-3, atol=5e-4 * max(1.0, float(want.abs().max())))
    for i in range(2):
        summed = sum(run1[0][r][1][i] for r in range(world))
        assert float((summed - params[i].grad.cpu()).norm() / params[i].grad.cpu().norm().clamp(min=1e-6)) < 1e-3
