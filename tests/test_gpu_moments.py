"""The moment aggregators on the GPU: the dense layer against the reference's own output and autograd (tests/golden/
dense_moments.pt), the kernels against float64 (tests/moment_bars.py) and the C oracle, bit-reproducibility, training, and
the multi-GPU planes with moments in the list (W ranks in one process, as in tests/test_gpu_halo_grad.py)."""
import pytest
import torch

from conftest import load_golden
import moment_oracle as MO
import moment_bars as MB

pytestmark = pytest.mark.gpu

S3 = ["identity", "amplification", "attenuation"]
AM = ["mean", "moment3", "max", "moment4", "moment5"]


def dev():
    return torch.device("cuda:0")


def zipf_graph(n, e, seed, hub=0):
    g = torch.Generator().manual_seed(seed)
    w = 1.0 / torch.arange(1, n + 1, dtype=torch.float64) ** 1.1
    dst = torch.multinomial(w, e, replacement=True, generator=g)
    src = torch.randint(0, n, (e,), generator=g)
    if hub:
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.full((hub,), 7)])
    return src, dst


def uniform_graph(n, e, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n, (e,), generator=g), torch.randint(0, int(n * 0.95), (e,), generator=g)


def test_dense_layer_matches_the_reference_forward_and_backward():
    import pna_b200
    g = load_golden("dense_moments")
    lay = pna_b200.dense.PNALayer(aggregators=g["aggregators"], scalers=g["scalers"], avg_d=g["avg_d"], **g["ctor"])
    lay.load_state_dict(g["state_dict"])
    lay = lay.to(dev()).eval()
    adj = g["adj"].to(dev())
    with torch.no_grad():
        out = lay(g["h"].to(dev()), adj).cpu()
    err = (out - g["out"]).abs().reshape(-1, out.size(-1))
    tol = _dense_out_bar(g, lay)
    assert (err <= tol).all(), float((err / tol).max())
    h = g["h"].to(dev()).requires_grad_(True)
    lay.zero_grad()
    (lay(h, adj) * g["grads"]["w"].to(dev())).sum().backward()
    torch.testing.assert_close(h.grad.cpu(), g["grads"]["h"], rtol=1e-3, atol=5e-4)
    for k, p in lay.named_parameters():
        ref = g["grads"]["params"][k]
        err = float((p.grad.cpu() - ref).norm() / ref.norm().clamp(min=1e-6))
        assert err < 2e-3, f"{k}: {err:.2e}"


def _dense_out_bar(g, lay):
    """The moment bar (tests/moment_bars.py) of the aggregate, carried through the post-MLP and the mixing layer (both
    Lipschitz with |W|), plus 2e-5 for the other columns and the fp32 GEMMs."""
    h, adj = g["h"], g["adj"]
    B, N, F = h.shape
    it, A, S = lay.input_tower, len(lay.aggregators), len(lay.scalers)
    b, i, j = (adj != 0).nonzero(as_tuple=True)
    dst, src, n = b * N + i, b * N + j, B * N
    hf = h.reshape(n, F)
    D = (adj != 0).sum(-1).reshape(n).double()
    lg = torch.log(D + 1)
    fac = {"identity": torch.ones_like(D), "amplification": lg / lay.avg_d["log"],
           "attenuation": torch.where(D > 0, lay.avg_d["log"] / lg, torch.ones_like(D))}
    post = []
    for t, tw in enumerate(lay.towers):
        lin = tw.pretrans.fully_connected[0].linear
        W, bias = lin.weight.detach().cpu(), lin.bias.detach().cpu()
        ht = hf[:, t * it:(t + 1) * it]
        msg = ht[dst] @ W[:, :it].t() + ht[src] @ W[:, it:].t() + bias        # pretrans([h_v, h_u]), self first
        cols = torch.zeros(n, 1 + A * S, it, dtype=torch.float64)
        for a, name in enumerate(lay.aggregators):
            if name.startswith("moment"):
                _, tol = MB.moment_bar(msg, dst, n, int(name[-1]))
                for s_, sc in enumerate(lay.scalers):
                    cols[:, 1 + s_ * A + a] = tol * fac[sc].abs().unsqueeze(1)
        Wp = tw.posttrans.fully_connected[0].linear.weight.detach().cpu().double().abs()
        post.append(cols.reshape(n, -1) @ Wp.t())
    Wm = lay.mixing_network.linear.weight.detach().cpu().double().abs()
    return (torch.cat(post, 1) @ Wm.t()).float() + 2e-5


@pytest.mark.parametrize("shape,dtype", [("uniform", torch.float32), ("uniform", torch.bfloat16), ("zipf", torch.float32),
                                         ("zipf", torch.bfloat16)])
def test_kernel_within_the_bar_and_the_c_oracle(shape, dtype):
    import pna_b200
    if shape == "uniform":      # config-2-like: ~10 in-edges per row, no split rows
        n, f = 20000, 64
        src, dst = uniform_graph(n, 10 * n, seed=2)
    else:                       # power law with split rows, one of them with more than 512 chunks
        n, f = 6000, 32
        src, dst = zipf_graph(n, 60000, seed=5, hub=70000)
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(n, f, generator=g) + 0.3).to(dtype)
    rb = torch.randn(n, f, generator=g).to(dtype)
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    if shape == "zipf":
        assert csr.n_hubs > 0 and csr.max_degree > 512 * csr.chunk_edges
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    out = pna_b200.aggregate_forward(x.to(dev()), csr, AM, S3, avg, row_bias=rb.to(dev())).float().cpu()
    again = pna_b200.aggregate_forward(x.to(dev()), csr, AM, S3, avg, row_bias=rb.to(dev())).float().cpu()
    assert torch.equal(out, again)
    msg = x.float()[src] + rb.float()[dst]
    deg = torch.bincount(dst, minlength=n)
    light = deg < csr.split_threshold
    ei = torch.stack([torch.arange(msg.size(0)), dst])
    A = len(AM)
    for a, name in enumerate(AM):
        if not name.startswith("moment"):
            continue
        k = int(name[-1])
        got = out[:, a * f:(a + 1) * f]                              # identity scaler
        r64, tol = MB.moment_bar(msg, dst, n, k)
        if dtype == torch.bfloat16:
            tol = tol + r64.abs() * 2.0 ** -8                         # the bf16 store
        assert ((got.double() - r64).abs() <= tol).all(), (name, float(((got.double() - r64).abs() / tol).max()))
        want = MO.moment(msg, ei, n, k)
        if dtype == torch.bfloat16:
            want = want.to(torch.bfloat16).float()
        # light rows: the C oracle's order; only the device powf differs (a few ulp), then the bf16 store
        ulp = 2.0 ** -23 if dtype == torch.float32 else 2.0 ** -7
        assert ((got[light] - want[light]).abs() <= 4 * ulp * want[light].abs()).all(), name
        assert torch.isfinite(out[:, (A + a) * f:(A + a + 1) * f]).all()


def _train_step_grads(dtype, mode, monkeypatch, deterministic):
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", mode)
    n, f = 5000, 48
    src, dst = zipf_graph(n, 40000, seed=9, hub=3000)
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(n, f, generator=g)).to(dtype).to(dev()).requires_grad_(True)
    rb = torch.randn(n, f, generator=g).to(dtype).to(dev()).requires_grad_(True)
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    w = torch.randn(n, 2 * len(AM) * 3 * f // 2, generator=g).to(dev())
    torch.use_deterministic_algorithms(deterministic)
    try:
        out = pna_b200.pna_aggregate(x, csr, AM, S3, avg, towers=2, row_bias=rb)
        (out.float() * w).sum().backward()
    finally:
        torch.use_deterministic_algorithms(False)
    return out.detach(), x.grad.clone(), rb.grad.clone()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_deterministic_mode_repeats_bit_for_bit_and_agrees_with_atomic(dtype, monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    o1, gx1, gb1 = _train_step_grads(dtype, "atomic", monkeypatch, True)
    o2, gx2, gb2 = _train_step_grads(dtype, "atomic", monkeypatch, True)
    assert torch.equal(o1, o2) and torch.equal(gx1, gx2) and torch.equal(gb1, gb2)
    for mode in ("atomic", "coef"):          # coef falls back to the atomic path for moments
        o3, gx3, gb3 = _train_step_grads(dtype, mode, monkeypatch, False)
        assert torch.equal(o1, o3)
        rel = 1e-4 if dtype == torch.float32 else 2e-2
        for a, b in ((gx1, gx3), (gb1, gb3)):   # same terms; the atomic mode adds them in run-dependent order
            assert float((a.float() - b.float()).abs().max()) <= rel * float(a.float().abs().max())


def test_multitask_stack_with_moments_trains():
    """A multitask-shaped model (dense layers over [B, N, F] with adj, the reference's GNN stack) learns a target."""
    import pna_b200
    torch.manual_seed(0)
    B, N, F = 16, 20, 16
    adj = (torch.rand(B, N, N) < 0.25).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float()
    for b in range(B):
        for i in range(N):
            if adj[b, i].sum() == 0:
                adj[b, i, (i + 1) % N] = adj[b, (i + 1) % N, i] = 1
    h = torch.randn(B, N, F)
    target = torch.einsum("bij,bjf->bif", adj, h).pow(2).mean(-1, keepdim=True)   # a neighbourhood statistic
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    aggrs = ["mean", "max", "moment3", "moment4", "std"]
    layers = torch.nn.ModuleList([pna_b200.dense.PNALayer(F, F, aggrs, S3, avg_d, towers=2, self_loop=False)
                                  for _ in range(2)]).to(dev())
    head = torch.nn.Linear(F, 1).to(dev())
    opt = torch.optim.Adam(list(layers.parameters()) + list(head.parameters()), lr=3e-3)
    adj, h, target = adj.to(dev()), h.to(dev()), target.to(dev())
    losses = []
    for _ in range(60):
        z = h
        for lay in layers:
            z = torch.relu(lay(z, adj))
        loss = torch.nn.functional.mse_loss(head(z), target)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(l == l for l in losses) and losses[-1] < 0.5 * losses[0], losses[::10]


def test_pull_plane_two_ranks_with_moments(monkeypatch):
    import pna_b200
    from test_gpu_halo_grad import _graph, _ranks
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    n, f, world = 1500, 64, 2
    src, dst = _graph(n, 10000, 800, seed=4)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, f, generator=g)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    w = torch.randn(n, len(AM) * 3 * f, generator=g).to(dev())
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    xg = x.to(dev()).requires_grad_(True)
    out = pna_b200.pna_aggregate(xg, csr, AM, S3, avg)
    (out * w).sum().backward()
    bounds, plans, aggs = _ranks(src, dst, n, f, world, torch.float32)
    xl = [x[int(bounds[r]):int(bounds[r + 1])].to(dev()) for r in range(world)]
    for r in range(world):
        aggs[r].x_local.copy_(xl[r])
    exts = [aggs[r].exchange_features(xl[r]).requires_grad_(True) for r in range(world)]
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        o = pna_b200.pna_aggregate(exts[r], aggs[r].csr, AM, S3, avg)
        assert torch.equal(o, out[lo:hi].detach())
        (o * w[lo:hi]).sum().backward()
    for r in range(world):
        aggs[r].stage_halo_grad(exts[r].grad)
    got = torch.cat([aggs[r].pull_halo_grad(exts[r].grad) for r in range(world)]).cpu()
    want = xg.grad.cpu()
    assert sum(p.n_halo for p in plans) > 0
    assert float((got - want).abs().max()) <= 1e-4 * float(want.abs().max())


def test_halo_plane_overlapped_forward_with_moments():
    import pna_b200
    from pna_b200 import dist as pd
    from test_gpu_halo_grad import _graph
    from test_gpu_halo_plane_grad import _on_device, _on_threads
    from test_halo_plane_grad_cpu import ThreadedAllToAll, halo_plans
    n, f, world = 1500, 64, 2
    src, dst = _graph(n, 10000, 800, seed=6)
    x = torch.randn(n, f, generator=torch.Generator().manual_seed(6))
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    out = pna_b200.aggregate_forward(x.to(dev()), csr, AM, S3, avg)
    bounds = pd.partition_bounds(torch.bincount(dst, minlength=n), world)
    plans = [_on_device(p) for p in halo_plans(src, dst, bounds, world)]
    a2a = ThreadedAllToAll(world)
    aggs = [pd.HaloAggregator(plans[r], f, group=r, overlap=True, _all_to_all=a2a) for r in range(world)]

    def rank(r):
        aggs[r].x_local.copy_(x[int(bounds[r]):int(bounds[r + 1])].to(dev()))
        o = aggs[r].aggregate(AM, S3, avg)
        torch.cuda.synchronize()
        return o
    res = _on_threads(world, rank, abort=[a2a.abort])
    assert sum(p.n_halo for p in plans) > 0
    for r in range(world):
        assert torch.equal(res[r], out[int(bounds[r]):int(bounds[r + 1])]), f"rank {r}"
