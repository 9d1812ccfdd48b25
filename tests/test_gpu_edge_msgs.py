"""The DGL PNALayer and the PyG PNAConv with edge features and / or more than one pretrans layer on the GPU, their messages
from pna_edge_msg_fwd / pna_edge_msg_bwd: against the reference's own outputs and autograd (tests/golden/dgl_edge_msgs*.pt,
tests/golden/pyg_edge_msgs.pt), the routing between the kernel and the torch message path, bit-reproducible training
steps, and a training run at the ZINC shape."""
import pytest
import torch

from conftest import load_golden

pytestmark = pytest.mark.gpu

DGL_CASES = ([("dgl_edge_msgs", f"L{L}_div{d}") for L in (1, 2, 3) for d in (1, 0)] +
             [("dgl_edge_msgs_zinc", "zinc"), ("dgl_edge_msgs_wide75", "wide75")])
PYG_CASES = [f"edge_L{L}_div{d}" for L in (1, 2, 3) for d in (1, 0)] + ["noedge_L3"]


def dev():
    return torch.device("cuda:0")


def _dgl_layer(g, c):
    import pna_b200
    lay = pna_b200.PNALayer(aggregators=c["aggregators"], scalers=c["scalers"], avg_d=c["avg_d"], **c["ctor"])
    lay.load_state_dict(c["state_dict"], strict=True)
    lay = lay.to(dev()).eval()
    ei = g["edge_index"]
    graph = pna_b200.Graph(ei[0], ei[1], c["h"].size(0)).to(dev())
    snorm = c["snorm_n"].to(dev())
    return lay, (lambda h, e: lay(graph, h, e, snorm)), [c["h"], c["e"]]


def _pyg_layer(g, c):
    import pna_b200
    k = c["ctor"]
    lay = pna_b200.PNAConv(aggregators=c["aggregators"], scalers=c["scalers"], deg=c["deg"], **k)
    lay.load_state_dict(c["state_dict"], strict=True)
    lay = lay.to(dev())
    ei = g["edge_index"].to(dev())
    return lay, (lambda x, ea: lay(x, ei, ea)), [c["x"], c["edge_attr"]]


def _check_case(make, fixture, name):
    g = load_golden(fixture)
    c = g["cases"][name]
    lay, call, inputs = make(g, c)
    with torch.no_grad():
        out = call(*[None if t is None else t.to(dev()) for t in inputs]).cpu()
    ref64 = c["out64"]
    # 1e-5 + 1e-5 |ref| from float64; where the reference's own fp32 output is further off, 2.5x its error
    bar = torch.maximum(1e-5 + 1e-5 * ref64.abs(), 2.5 * (c["out"].double() - ref64).abs())
    err = (out.double() - ref64).abs()
    assert (err <= bar).all(), float((err / bar).max())
    ins = [None if t is None else t.to(dev()).requires_grad_(True) for t in inputs]
    lay.zero_grad()
    (call(*ins) * c["w"].to(dev())).sum().backward()
    for t, want in zip(ins, c["input_grads"]):                # x / h, and edge_attr / e: the reference's fp32 autograd
        if t is not None:
            torch.testing.assert_close(t.grad.cpu(), want, rtol=1e-3, atol=5e-4)
    for k, p in lay.named_parameters():
        # against the float64 gradient (stored rounded to fp32: 6e-8 relative, far below the bar); where the reference's own
        # fp32 gradient is further than 2e-3 from it, 2.5x that error is the bar
        ref = c["params64"][k].double()
        err = float((p.grad.cpu().double() - ref).norm() / ref.norm().clamp(min=1e-6))
        ref_err = c["ref_err"][k]
        assert err < max(2e-3, 2.5 * ref_err), f"{k}: {err:.2e} (reference fp32: {ref_err:.2e})"


def _no_torch_messages(monkeypatch):
    """Make the torch message paths of both layers raise: whatever passes ran its messages through the kernel (also in
    training steps on these small graphs)."""
    import pna_b200
    monkeypatch.setattr(pna_b200.edge_mlp, "FUSED_TRAINING_MIN_EDGES", 0)

    def boom(*a, **k):
        raise AssertionError("torch message path taken")
    monkeypatch.setattr(pna_b200.dgl_layers.PNALayer, "_edge_messages", boom)
    monkeypatch.setattr(pna_b200.pyg.PNAConv, "_messages_in_slot_order", boom)


@pytest.mark.parametrize("fixture,name", DGL_CASES)
def test_dgl_layer_matches_the_reference_through_the_kernel(fixture, name, monkeypatch):
    _no_torch_messages(monkeypatch)
    _check_case(_dgl_layer, fixture, name)


@pytest.mark.parametrize("name", PYG_CASES)
def test_pyg_conv_matches_the_reference_through_the_kernel(name, monkeypatch):
    _no_torch_messages(monkeypatch)
    _check_case(_pyg_layer, "pyg_edge_msgs", name)


def _small_graph(n=300, e=1500, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g), n


def test_inputs_the_kernel_does_not_take_reach_the_torch_path(monkeypatch):
    """bf16, and pretrans_layers >= 2 at a tower width above 64, build their messages in torch; the kernel is not called."""
    import pna_b200
    from pna_b200 import dgl_layers, pyg

    def boom(*a, **k):
        raise AssertionError("edge message kernel called")
    monkeypatch.setattr(dgl_layers, "edge_messages", boom)
    monkeypatch.setattr(pyg, "edge_messages", boom)
    src, dst, n = _small_graph()
    ei = torch.stack([src, dst]).to(dev())
    deg = torch.bincount(torch.bincount(dst, minlength=n))
    conv = pna_b200.PNAConv(16, 16, ["mean", "max"], ["identity"], deg, edge_dim=4, towers=2, pre_layers=2,
                            divide_input=True).to(dev()).to(torch.bfloat16)
    x = torch.randn(n, 16, device=dev(), dtype=torch.bfloat16)
    out = conv(x, ei, torch.randn(src.numel(), 4, device=dev(), dtype=torch.bfloat16))
    assert out.dtype == torch.bfloat16 and bool(torch.isfinite(out.float()).all())
    avg = {"log": 1.5, "lin": 5.0}
    lay = pna_b200.PNALayer(66, 66, "mean max", "identity", avg, 0.0, False, False, towers=2, pretrans_layers=2,
                            divide_input=False, edge_features=True, edge_dim=3).to(dev())
    graph = pna_b200.Graph(src, dst, n).to(dev())
    out = lay(graph, torch.randn(n, 66, device=dev()), torch.randn(src.numel(), 3, device=dev()), None)
    assert out.shape == (n, 66) and bool(torch.isfinite(out).all())
    with pytest.raises(AssertionError, match="kernel called"), torch.no_grad():     # F_t = 33 with L = 2: the kernel's
        pna_b200.PNALayer(66, 66, "mean", "identity", avg, 0.0, False, False, towers=2, pretrans_layers=2, edge_features=True,
                          edge_dim=3).to(dev())(graph, torch.randn(n, 66, device=dev()), torch.randn(src.numel(), 3,
                                                                                                  device=dev()), None)


def test_small_training_steps_take_the_torch_path(monkeypatch):
    """Below FUSED_TRAINING_MIN_EDGES a step with autograd builds its messages in torch; the same call without autograd
    takes the kernel; both give the reference's output."""
    import pna_b200
    from pna_b200 import dgl_layers
    g = load_golden("dgl_edge_msgs")
    c = g["cases"]["L2_div1"]
    lay, call, (h, e) = _dgl_layer(g, c)
    assert g["edge_index"].size(1) < pna_b200.edge_mlp.FUSED_TRAINING_MIN_EDGES
    calls = []
    real = dgl_layers.edge_messages
    monkeypatch.setattr(dgl_layers, "edge_messages", lambda *a, **k: calls.append(1) or real(*a, **k))
    out = call(h.to(dev()).requires_grad_(True), e.to(dev()))
    assert not calls
    with torch.no_grad():
        out2 = call(h.to(dev()), e.to(dev()))
    assert calls
    torch.testing.assert_close(out.detach(), out2, rtol=1e-5, atol=1e-5)


def test_deterministic_training_steps_repeat_bit_for_bit(monkeypatch):
    import pna_b200
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    _no_torch_messages(monkeypatch)
    src, dst, n = _small_graph(seed=3)
    ei = torch.stack([src, dst]).to(dev())
    deg = torch.bincount(torch.bincount(dst, minlength=n))
    avg = {"log": 1.7, "lin": 5.0}
    gen = torch.Generator().manual_seed(4)
    h = torch.randn(n, 20, generator=gen).to(dev())
    e = torch.randn(src.numel(), 6, generator=gen).to(dev())
    torch.manual_seed(6)
    dgl = pna_b200.PNALayer(20, 20, "mean max min std", "identity amplification attenuation", avg, 0.0, True, True, towers=5,
                            pretrans_layers=2, edge_features=True, edge_dim=6).to(dev())
    conv = pna_b200.PNAConv(20, 20, ["mean", "min", "max", "std"], ["identity", "amplification"], deg, edge_dim=6, towers=2,
                            pre_layers=3, divide_input=True).to(dev())
    graph = pna_b200.Graph(src, dst, n).to(dev())
    snorm = torch.full((n, 1), n ** -0.5, device=dev())
    models = torch.nn.ModuleList([dgl, conv])
    opt = torch.optim.SGD(models.parameters(), lr=1e-2)

    def two_steps():
        state = {k: v.clone() for k, v in models.state_dict().items()}
        grads = []
        for _ in range(2):
            x, ea = h.clone().requires_grad_(True), e.clone().requires_grad_(True)
            opt.zero_grad()
            (dgl(graph, x, ea, snorm).pow(2).mean() + conv(x, ei, ea).pow(2).mean()).backward()
            grads.append([x.grad.clone(), ea.grad.clone()] + [p.grad.clone() for p in models.parameters()])
            opt.step()
        models.load_state_dict(state)
        return grads

    torch.use_deterministic_algorithms(True)
    try:
        g1, g2 = two_steps(), two_steps()
    finally:
        torch.use_deterministic_algorithms(False)
    for s1, s2 in zip(g1, g2):
        for a, b in zip(s1, s2):
            assert torch.equal(a, b)


def test_zinc_shaped_dgl_stack_with_edge_features_trains(monkeypatch):
    """Four DGL layers at the README's ZINC shape (hidden 70, towers 5, divide_input, edge_dim 50) learn a graph target."""
    import pna_b200
    from pna_b200 import synth
    _no_torch_messages(monkeypatch)
    ei, x, node_graph = synth.zinc_like(n_graphs=64, n_feat=70)
    n, G = x.size(0), 64
    gen = torch.Generator().manual_seed(1)
    e = torch.randn(ei.size(1), 50, generator=gen)
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    graph = pna_b200.Graph(ei[0], ei[1], n).to(dev())
    # a target that needs the edge features: per graph, the mean over edges of e[:, 0] times the source's first feature
    t = torch.zeros(G).index_add_(0, node_graph[ei[1]], e[:, 0] * x[ei[0], 0]) / torch.bincount(node_graph[ei[1]],
                                                                                                  minlength=G).clamp(min=1)
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([pna_b200.PNALayer(70, 70, "mean max min std", "identity amplification attenuation", avg, 0.0,
                                                    True, True, towers=5, divide_input=True, residual=True,
                                                    edge_features=True, edge_dim=50) for _ in range(4)]).to(dev())
    head = torch.nn.Linear(70, 1).to(dev())
    opt = torch.optim.Adam(list(layers.parameters()) + list(head.parameters()), lr=1e-3)
    x, e, t, ng = x.to(dev()), e.to(dev()), t.to(dev()), node_graph.to(dev())
    snorm = torch.ones(n, 1, device=dev())
    losses = []
    for _ in range(60):
        z = x
        for lay in layers:
            z = lay(graph, z, e, snorm)
        pooled = torch.zeros(G, 70, device=dev()).index_add_(0, ng, z)
        loss = torch.nn.functional.mse_loss(head(pooled).squeeze(1), t)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert all(l == l for l in losses) and losses[-1] < 0.5 * losses[0], losses[::10]
