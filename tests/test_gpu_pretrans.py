"""The dense layer with pretrans_layers >= 2 on the GPU: against the reference's own output and autograd
(tests/golden/dense_pretrans.pt), the edge-MLP messages against float64 and against the reference's fp32 error,
normalised_mean with degree_col against the gathered call, bit-reproducible training steps, and a training run."""
import pytest
import torch

from conftest import load_golden
import moment_bars as MB
import weighted_bars as WB
from test_gpu_moments import S3, dev

pytestmark = pytest.mark.gpu

WEIGHTED = ("softmax", "softmin", "normalised_mean")
CASES = [f"L{L}_div{d}_loop{s}_{g}" for L in (2, 3) for d in (1, 0) for s in (0, 1) for g in ("plain", "addon")]


def _mlp(m, x):
    """The pretrans MLP as the reference evaluates it (nn.Linear, ReLU between layers), in x's dtype and on x's device."""
    fcs = m.fully_connected
    for k, fc in enumerate(fcs):
        x = torch.nn.functional.linear(x, fc.linear.weight.detach().to(x), fc.linear.bias.detach().to(x))
        if k < len(fcs) - 1:
            x = torch.relu(x)
    return x


def _tower_inputs(h, lay, t):
    it = lay.input_tower
    return h[:, t * it:(t + 1) * it] if lay.divide_input else h


def _dense_out_bar(g, lay, self_loop, ref):
    """1e-5 + 1e-5 |ref| for the plain aggregators; the moment and weighted columns' bars (tests/moment_bars.py,
    tests/weighted_bars.py, on float64 messages of the same pretrans MLP) carried through the post-MLP and the mixing
    layer with |W|, plus 2e-5."""
    h, adj = g["h"].double(), g["adj"]
    B, N, F = h.shape
    a = adj + torch.eye(N).unsqueeze(0) if self_loop else adj
    A, S = len(lay.aggregators), len(lay.scalers)
    b, i, j = (a != 0).nonzero(as_tuple=True)
    dst, src, n = b * N + i, b * N + j, B * N
    hf = h.reshape(n, F)
    D = (adj != 0).sum(-1).reshape(n).double()
    lg = torch.log(D + 1)
    fac = {"identity": torch.ones_like(D), "amplification": lg / lay.avg_d["log"],
           "attenuation": torch.where(D > 0, lay.avg_d["log"] / lg, torch.ones_like(D))}
    post = []
    for t, tw in enumerate(lay.towers):
        ht = _tower_inputs(hf, lay, t)
        msg = _mlp(tw.pretrans, torch.cat([ht[dst], ht[src]], 1))            # pretrans([h_v, h_u]), self first
        cols = torch.zeros(n, 1 + A * S, lay.input_tower, dtype=torch.float64)
        for a_, name in enumerate(lay.aggregators):
            tol = None
            if name in WEIGHTED:
                _, tol = WB.bar(name, msg, dst, n, wsrc=src)
            elif name.startswith("moment"):
                _, tol = MB.moment_bar(msg, dst, n, int(name[-1]))
            if tol is not None:
                for s_, sc in enumerate(lay.scalers):
                    cols[:, 1 + s_ * A + a_] = tol * fac[sc].abs().unsqueeze(1)
        Wp = tw.posttrans.fully_connected[0].linear.weight.detach().cpu().double().abs()
        post.append(cols.reshape(n, -1) @ Wp.t())
    Wm = lay.mixing_network.linear.weight.detach().cpu().double().abs()
    carried = (torch.cat(post, 1) @ Wm.t()).float()
    return 1e-5 + 1e-5 * ref.abs().reshape(n, -1) + carried + 2e-5 * (carried > 0)


@pytest.mark.parametrize("name", CASES)
def test_dense_layer_matches_the_reference_forward_and_backward(name):
    import pna_b200
    g = load_golden("dense_pretrans")
    case = g["cases"][name]
    lay = pna_b200.dense.PNALayer(aggregators=case["aggregators"], scalers=g["scalers"], avg_d=case["avg_d"], **case["ctor"])
    lay.load_state_dict(case["state_dict"], strict=True)
    tol = _dense_out_bar(g, lay, case["ctor"]["self_loop"], case["out64"].float())
    lay = lay.to(dev()).eval()
    adj = g["adj"].to(dev())
    with torch.no_grad():
        out = lay(g["h"].to(dev()), adj).cpu()
    for want in (case["out"], case["out64"].float()):
        err = (out - want).abs().reshape(-1, out.size(-1))
        assert (err <= tol).all(), float((err / tol).max())
    h = g["h"].to(dev()).requires_grad_(True)
    lay.zero_grad()
    (lay(h, adj) * case["grads"]["w"].to(dev())).sum().backward()
    torch.testing.assert_close(h.grad.cpu(), case["grads"]["h"], rtol=1e-3, atol=5e-4)
    for k, p in lay.named_parameters():
        ref = case["grads64"]["params"][k]
        norm = ref.norm().clamp(min=1e-6)
        err = float((p.grad.cpu().double() - ref).norm() / norm)
        # where the reference's own fp32 gradient is further than 2e-3 from float64 (L = 3 with var / std: rows whose
        # messages nearly coincide sit on the kink of relu(var) and the steep sqrt of std), 2.5x its error is the bar
        ref_err = float((case["grads"]["params"][k].double() - ref).norm() / norm)
        assert err < max(2e-3, 2.5 * ref_err), f"{k}: {err:.2e} (reference fp32: {ref_err:.2e})"


def _graph_with_split_rows(n, seed):
    """Uniform sources, ~8 in-edges per row, and five rows with 300 .. 700 in-edges (above the split threshold)."""
    g = torch.Generator().manual_seed(seed)
    dst = torch.randint(0, n, (8 * n,), generator=g)
    hubs = torch.cat([torch.full((300 + 100 * k,), 3 + 17 * k) for k in range(5)])
    dst = torch.cat([dst, hubs])
    src = torch.randint(0, n, (dst.numel(),), generator=g)
    return src, dst


@pytest.mark.parametrize("L,Ft,T", [(2, 8, 2), (3, 16, 2), (4, 64, 1), (3, 5, 3)])
def test_messages_within_the_bar_and_the_reference_fp32_error(L, Ft, T):
    import pna_b200
    from pna_b200.edge_mlp import edge_mlp
    from pna_b200.nn_blocks import MLP
    n = 4000
    src, dst = _graph_with_split_rows(n, seed=L * 100 + Ft)
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    assert int(csr.in_degree.max()) >= 256 and csr.n_hubs >= 1
    torch.manual_seed(Ft + T)
    h = torch.randn(n, T * Ft)
    mlps = [MLP(2 * Ft, Ft, Ft, L, mid_activation="relu", last_activation="none") for _ in range(T)]
    for m in mlps:
        for fc in m.fully_connected:
            torch.nn.init.normal_(fc.linear.weight, std=1.0 / Ft ** 0.5)
            torch.nn.init.normal_(fc.linear.bias, std=0.3)
    i, j = csr.dst_of_slot.cpu(), csr.col.long().cpu()
    E = csr.n_edges
    # the kernel's inputs, and the messages in float64 from the same inputs
    W1 = [m.fully_connected[0].linear for m in mlps]
    hs = [h[:, t * Ft:(t + 1) * Ft] for t in range(T)]
    A = torch.cat([hs[t] @ W1[t].weight[:, :Ft].t() for t in range(T)], 1).detach()
    Bm = torch.cat([hs[t] @ W1[t].weight[:, Ft:].t() for t in range(T)], 1).detach()
    b1 = torch.cat([l.bias for l in W1]).detach()
    W = torch.stack([torch.stack([m.fully_connected[k].linear.weight for m in mlps]) for k in range(1, L)]).detach()
    bW = torch.stack([torch.stack([m.fully_connected[k].linear.bias for m in mlps]) for k in range(1, L)]).detach()
    M = edge_mlp(A.to(dev()), Bm.to(dev()), b1.to(dev()), W.to(dev()), bW.to(dev()), csr, T).cpu().double()
    z = torch.relu(A.double()[i] + Bm.double()[j] + b1.double())
    c = A.double().abs()[i] + Bm.double().abs()[j] + b1.double().abs()
    for k in range(2, L + 1):
        u = torch.einsum("toc,etc->eto", W[k - 2].double(), z.view(E, T, Ft)).reshape(E, -1) + bW[k - 2].double().reshape(-1)
        z = u if k == L else torch.relu(u)
        c = torch.einsum("toc,etc->eto", W[k - 2].double().abs(), c.view(E, T, Ft)).reshape(E, -1) + \
            bW[k - 2].double().abs().reshape(-1)
    bar = (Ft + 2) * L * 2.0 ** -24 * c
    assert ((M - z).abs() <= bar).all(), float(((M - z).abs() / bar).max())
    # end to end from h: this library (node GEMMs + kernel) against the reference's fp32 pretrans on [h_i, h_j]
    with torch.no_grad():
        pair = [torch.cat([hs[t][i], hs[t][j]], 1) for t in range(T)]
        ref32 = torch.cat([_mlp(mlps[t], pair[t].to(dev())).cpu() for t in range(T)], 1).double()
        ref64 = torch.cat([_mlp(mlps[t], pair[t].double()) for t in range(T)], 1)
    err_ours, err_ref = float((M - ref64).norm()), float((ref32 - ref64).norm())
    assert err_ours <= 2.5 * err_ref, (err_ours, err_ref)


def test_normalised_mean_with_degree_col_is_the_gathered_call(monkeypatch):
    """x[col] in slot order with degree_col = col gives the bits of the gathered call: the forward, the deterministic
    backward (per-slot gradients summed over the slot-transposed CSR) and the atomic backward's per-slot gradients."""
    import pna_b200
    from pna_b200 import aggregate as agg
    n, F = 3000, 24
    src, dst = _graph_with_split_rows(n, seed=7)
    csr = pna_b200.build_csr(src.to(dev()), dst.to(dev()), n)
    assert csr.n_hubs >= 1
    g = torch.Generator().manual_seed(3)
    x = torch.randn(n, F, generator=g).to(dev())
    rb = torch.randn(n, F, generator=g).to(dev())
    xs = x[csr.col.long()].contiguous()
    avg = {"log": 2.0, "lin": 8.0}
    kw = dict(towers=2, row_bias=rb)
    names = ["normalised_mean"]
    o1 = agg.aggregate_forward(x, csr, names, S3, avg, **kw)
    o2 = agg.aggregate_forward(xs, csr, names, S3, avg, messages_in_csr_order=True, degree_col=csr.col, **kw)
    assert torch.equal(o1, o2)
    go = torch.randn(o1.shape, generator=g).to(dev())
    bkw = dict(towers=2, row_bias=rb, need_bias_grad=True)
    torch.use_deterministic_algorithms(True)
    try:
        gx, gb = agg.aggregate_backward(go, x, csr, names, S3, avg, **bkw)
        gs, gb2 = agg.aggregate_backward(go, xs, csr, names, S3, avg, messages_in_csr_order=True, degree_col=csr.col, **bkw)
    finally:
        torch.use_deterministic_algorithms(False)
    summed = agg.aggregate_forward(gs, csr.slot_transposed(n), ["sum"], ["identity"], {"log": 1.0, "lin": 1.0})
    assert torch.equal(gx, summed) and torch.equal(gb, gb2)
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    gs3, gb3 = agg.aggregate_backward(go, xs, csr, names, S3, avg, messages_in_csr_order=True, degree_col=csr.col, **bkw)
    _, gb4 = agg.aggregate_backward(go, x, csr, names, S3, avg, **bkw)
    assert torch.equal(gs3, gs) and torch.equal(gb3, gb) and torch.equal(gb4, gb)


def _adjacency(B, N, seed, p=0.25):
    torch.manual_seed(seed)
    adj = (torch.rand(B, N, N) < p).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float()
    for b in range(B):
        for i in range(N):
            if adj[b, i].sum() == 0:
                adj[b, i, (i + 1) % N] = adj[b, (i + 1) % N, i] = 1
    return adj


def test_deterministic_training_steps_repeat_bit_for_bit(monkeypatch):
    import pna_b200
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    B, N, F = 8, 20, 16
    adj = _adjacency(B, N, 1).to(dev())
    h = torch.randn(B, N, F, generator=torch.Generator().manual_seed(2)).to(dev())
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    aggrs = ["mean", "max", "softmax", "normalised_mean", "moment3", "identity"]
    torch.manual_seed(5)
    lay = pna_b200.dense.PNALayer(F, F, aggrs, S3, avg_d, towers=2, pretrans_layers=3).to(dev())
    opt = torch.optim.SGD(lay.parameters(), lr=1e-2)

    def two_steps():
        state = {k: v.clone() for k, v in lay.state_dict().items()}
        grads = []
        for _ in range(2):
            x = h.clone().requires_grad_(True)
            opt.zero_grad()
            lay(x, adj).pow(2).mean().backward()
            grads.append([x.grad.clone()] + [p.grad.clone() for p in lay.parameters()])
            opt.step()
        lay.load_state_dict(state)
        return grads

    torch.use_deterministic_algorithms(True)
    try:
        g1, g2 = two_steps(), two_steps()
    finally:
        torch.use_deterministic_algorithms(False)
    for s1, s2 in zip(g1, g2):
        for a, b in zip(s1, s2):
            assert torch.equal(a, b)


def test_multitask_stack_with_pretrans_layers_2_trains():
    """A four-layer multitask-shaped model (dense layers over [B, N, F] with adj, pretrans_layers=2) learns a target."""
    import pna_b200
    B, N, F = 16, 20, 16
    adj = _adjacency(B, N, 0)
    h = torch.randn(B, N, F)
    target = torch.einsum("bij,bjf->bif", adj, h).pow(2).mean(-1, keepdim=True)   # a neighbourhood statistic
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    aggrs = ["mean", "max", "min", "std"]
    layers = torch.nn.ModuleList([pna_b200.dense.PNALayer(F, F, aggrs, S3, avg_d, towers=2, pretrans_layers=2,
                                                          self_loop=(k % 2 == 1)) for k in range(4)]).to(dev())
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
