"""softmax / softmin / normalised_mean / identity on the GPU: the dense layer against the reference's own output and
autograd (tests/golden/dense_weighted.pt), the kernels against float64 (tests/weighted_bars.py) and the C oracle,
bit-reproducibility, training, and the pull plane with softmax / softmin in the list (two ranks in one process, as in
tests/test_gpu_moments.py)."""
import pytest
import torch

from conftest import load_golden
import weighted_bars as WB
import weighted_oracle as WO
from test_gpu_moments import S3, dev, uniform_graph, zipf_graph

pytestmark = pytest.mark.gpu

AW = ["mean", "softmax", "max", "softmin", "normalised_mean"]
WEIGHTED = ("softmax", "softmin", "normalised_mean")


@pytest.mark.parametrize("self_loop", [False, True])
def test_dense_layer_matches_the_reference_forward_and_backward(self_loop):
    import pna_b200
    g = load_golden("dense_weighted")
    case = g["cases"][str(self_loop)]
    lay = pna_b200.dense.PNALayer(aggregators=g["aggregators"], scalers=g["scalers"], avg_d=case["avg_d"], **case["ctor"])
    lay.load_state_dict(case["state_dict"])
    lay = lay.to(dev()).eval()
    adj = g["adj"].to(dev())
    with torch.no_grad():
        out = lay(g["h"].to(dev()), adj).cpu()
    tol = _dense_out_bar(g, lay, self_loop)
    for want in (case["out"], case["out64"].float()):
        err = (out - want).abs().reshape(-1, out.size(-1))
        assert (err <= tol).all(), float((err / tol).max())
    h = g["h"].to(dev()).requires_grad_(True)
    lay.zero_grad()
    (lay(h, adj) * case["grads"]["w"].to(dev())).sum().backward()
    torch.testing.assert_close(h.grad.cpu(), case["grads"]["h"], rtol=1e-3, atol=5e-4)
    for k, p in lay.named_parameters():
        ref = case["grads64"]["params"][k]
        err = float((p.grad.cpu().double() - ref).norm() / ref.norm().clamp(min=1e-6))
        assert err < 2e-3, f"{k}: {err:.2e}"


def _dense_out_bar(g, lay, self_loop):
    """The bars of tests/weighted_bars.py on the aggregate, carried through the post-MLP and the mixing layer (both
    Lipschitz with |W|), plus 2e-5 for the other columns (identity included) and the fp32 GEMMs."""
    h, adj = g["h"], g["adj"]
    B, N, F = h.shape
    a = adj + torch.eye(N).unsqueeze(0) if self_loop else adj
    it, A, S = lay.input_tower, len(lay.aggregators), len(lay.scalers)
    b, i, j = (a != 0).nonzero(as_tuple=True)
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
        for a_, name in enumerate(lay.aggregators):
            if name in WEIGHTED:
                _, tol = WB.bar(name, msg, dst, n, wsrc=src)
                for s_, sc in enumerate(lay.scalers):
                    cols[:, 1 + s_ * A + a_] = tol * fac[sc].abs().unsqueeze(1)
        Wp = tw.posttrans.fully_connected[0].linear.weight.detach().cpu().double().abs()
        post.append(cols.reshape(n, -1) @ Wp.t())
    Wm = lay.mixing_network.linear.weight.detach().cpu().double().abs()
    return (torch.cat(post, 1) @ Wm.t()).float() + 2e-5


def _column(out, n, towers, Ft, has_self, A, s, a, t):
    W = out.size(1) // towers
    base = t * W + (Ft if has_self else 0) + (s * A + a) * Ft
    return out[:, base:base + Ft]


@pytest.mark.parametrize("shape,dtype,towers,self_feat,sdeg", [
    ("uniform", torch.float32, 1, False, False), ("uniform", torch.bfloat16, 2, True, True),
    ("zipf", torch.float32, 2, True, False), ("zipf", torch.bfloat16, 1, False, True)])
def test_kernel_within_the_bar_and_the_c_oracle(shape, dtype, towers, self_feat, sdeg):
    import pna_b200
    if shape == "uniform":      # config-2-like: ~10 in-edges per row, no split rows
        n, f = 20000, 64
        src, dst = uniform_graph(n, 10 * n, seed=2)
    else:                       # power law with split rows, one of them with more than 512 chunks
        n, f = 6000, 32
        src, dst = zipf_graph(n, 60000, seed=5, hub=70000)
    g = torch.Generator().manual_seed(11)
    x = (torch.randn(n, f, generator=g) * 2 + 0.3).to(dtype)
    rb = torch.randn(n, f, generator=g).to(dtype)
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    if shape == "zipf":
        assert csr.n_hubs > 0 and csr.max_degree > 512 * csr.chunk_edges
    deg = torch.bincount(dst, minlength=n)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    kw = dict(towers=towers, row_bias=rb.to(dev()))
    if self_feat:
        kw["self_feat"] = x.to(dev())
    sd = (deg + torch.arange(n) % 3).to(torch.int32) if sdeg else deg
    if sdeg:
        kw["scaler_degree"] = sd.to(dev())
    out = pna_b200.aggregate_forward(x.to(dev()), csr, AW, S3, avg, **kw).float().cpu()
    again = pna_b200.aggregate_forward(x.to(dev()), csr, AW, S3, avg, **kw).float().cpu()
    assert torch.equal(out, again)
    msg = x.float()[src] + rb.float()[dst]
    light = deg < csr.split_threshold
    Ft, A = f // towers, len(AW)
    lg = torch.log(sd.double() + 1)
    for a, name in enumerate(AW):
        if name not in WEIGHTED:
            continue
        y64, tol = WB.bar(name, msg, dst, n, wsrc=src)
        want = WO.weighted(msg, dst, n, name, wsrc=src)
        if name == "normalised_mean":
            slack = want.abs().double()
        else:       # the device expf (2 ulp) against the host's: each e_s moves y by p_s (n_s - y') times its error
            nn_, _, _, p, yp = WB._softmax_parts(msg, dst, n, -1.0 if name == "softmin" else 1.0)
            slack = want.abs().double() + torch.zeros_like(yp).index_add(0, dst, p * (nn_ - yp[dst]).abs())
        if dtype == torch.bfloat16:
            tol = tol + y64.abs() * 2.0 ** -8                         # the bf16 store
            want = want.to(torch.bfloat16).float()
        ulp = 2.0 ** -23 if dtype == torch.float32 else 2.0 ** -7
        for t in range(towers):
            sl = slice(t * Ft, (t + 1) * Ft)
            got = _column(out, n, towers, Ft, self_feat, A, 0, a, t)
            err = (got.double() - y64[:, sl]).abs()
            assert (err <= tol[:, sl]).all(), (name, t, float((err / tol[:, sl]).max()))
            # light rows: the C oracle's order; only the device expf differs, then the bf16 store
            d = (got[light] - want[:, sl][light]).abs().double()
            assert (d <= 4 * ulp * slack[:, sl][light]).all(), (name, t)
            amp = _column(out, n, towers, Ft, self_feat, A, 1, a, t)
            torch.testing.assert_close(amp.double(), got.double() * (lg / avg["log"]).unsqueeze(1),
                                       rtol=1e-6 if dtype == torch.float32 else 2.0 ** -7, atol=0)
    assert torch.isfinite(out).all()


def _train_step_grads(dtype, mode, monkeypatch, deterministic):
    import pna_b200
    monkeypatch.setenv("PNA_B200_BWD", mode)
    n, f = 5000, 48
    src, dst = zipf_graph(n, 40000, seed=9, hub=3000)
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(n, f, generator=g)).to(dtype).to(dev()).requires_grad_(True)
    rb = torch.randn(n, f, generator=g).to(dtype).to(dev()).requires_grad_(True)
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    assert csr.n_hubs > 0
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    w = torch.randn(n, len(AW) * 3 * f, generator=g).to(dev())
    torch.use_deterministic_algorithms(deterministic)
    try:
        out = pna_b200.pna_aggregate(x, csr, AW, S3, avg, towers=2, row_bias=rb)
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
    for mode in ("atomic", "coef"):          # coef falls back to the atomic path for these aggregators
        o3, gx3, gb3 = _train_step_grads(dtype, mode, monkeypatch, False)
        assert torch.equal(o1, o3)
        rel = 1e-4 if dtype == torch.float32 else 2e-2
        for a, b in ((gx1, gx3), (gb1, gb3)):   # same terms; the atomic mode adds them in run-dependent order
            assert float((a.float() - b.float()).abs().max()) <= rel * float(a.float().abs().max())


def test_multitask_stack_with_the_new_aggregators_trains():
    """A four-layer multitask-shaped model (dense layers over [B, N, F] with adj) with every new name learns a target."""
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
    aggrs = ["mean", "softmax", "softmin", "normalised_mean", "identity", "max"]
    layers = torch.nn.ModuleList([pna_b200.dense.PNALayer(F, F, aggrs, S3, avg_d, towers=2, self_loop=(k % 2 == 1))
                                  for k in range(4)]).to(dev())
    head = torch.nn.Linear(F, 1).to(dev())
    opt = torch.optim.Adam(list(layers.parameters()) + list(head.parameters()), lr=3e-3)
    adj, h, target = adj.to(dev()), h.to(dev()), target.to(dev())
    losses = []
    for _ in range(80):
        z = h
        for lay in layers:
            z = torch.relu(lay(z, adj))
        loss = torch.nn.functional.mse_loss(head(z), target)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(l == l for l in losses) and losses[-1] < 0.5 * losses[0], losses[::10]


def test_pull_plane_two_ranks_with_softmax_and_softmin(monkeypatch):
    import pna_b200
    from test_gpu_halo_grad import _graph, _ranks
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    AS = ["mean", "softmax", "max", "softmin"]
    n, f, world = 1500, 64, 2
    src, dst = _graph(n, 10000, 800, seed=4)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(n, f, generator=g)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(torch.bincount(dst, minlength=n)))
    w = torch.randn(n, len(AS) * 3 * f, generator=g).to(dev())
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    xg = x.to(dev()).requires_grad_(True)
    out = pna_b200.pna_aggregate(xg, csr, AS, S3, avg)
    (out * w).sum().backward()
    bounds, plans, aggs = _ranks(src, dst, n, f, world, torch.float32)
    xl = [x[int(bounds[r]):int(bounds[r + 1])].to(dev()) for r in range(world)]
    for r in range(world):
        aggs[r].x_local.copy_(xl[r])
    exts = [aggs[r].exchange_features(xl[r]).requires_grad_(True) for r in range(world)]
    for r in range(world):
        lo, hi = int(bounds[r]), int(bounds[r + 1])
        o = pna_b200.pna_aggregate(exts[r], aggs[r].csr, AS, S3, avg)
        assert torch.equal(o, out[lo:hi].detach())
        if exts[r].size(0) != aggs[r].csr.n_nodes:                    # [local ; halo] rows have no local degree
            with pytest.raises(ValueError, match="normalised_mean"):
                pna_b200.pna_aggregate(exts[r], aggs[r].csr, ["normalised_mean"], S3, avg)
        (o * w[lo:hi]).sum().backward()
    for r in range(world):
        aggs[r].stage_halo_grad(exts[r].grad)
    got = torch.cat([aggs[r].pull_halo_grad(exts[r].grad) for r in range(world)]).cpu()
    want = xg.grad.cpu()
    assert sum(p.n_halo for p in plans) > 0
    assert float((got - want).abs().max()) <= 1e-4 * float(want.abs().max())
