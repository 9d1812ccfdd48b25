"""The tower post linear on the GPU: pna_linear_towers_scaled_fwd / pna_linear_towers_bwd_data against the exact restatement
(tests/towers_paths_ref.py) bit for bit on grid data and within its bars on random data; PNAConv and the DGL PNALayer take
the compact path and agree with the materialised path (PNA_B200_COMPACT_POST=0) forward and in every gradient; refused
shapes keep the materialised path; bit-reproducible training steps; and the memory a ZINC-shaped training step saves."""
import numpy as np
import pytest
import torch

import towers_paths_ref as R

pytestmark = pytest.mark.gpu


def dev():
    return torch.device("cuda:0")


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(dev())


@pytest.mark.parametrize("grid", [True, False], ids=["grid", "random"])
@pytest.mark.parametrize("case", R.CASES)
def test_kernels_match_the_restatement(case, grid):
    from pna_b200.linear import linear_towers_bwd_data, linear_towers_scaled_tf32x3
    n, t_n, fp, o, n_aggr, s_n = case
    a, c, w, b, gy = R.case_data(case, grid=grid)
    y = linear_towers_scaled_tf32x3(_t(a), _t(c), _t(w), _t(b)).cpu().numpy()
    ga = linear_towers_bwd_data(_t(gy), _t(c), _t(w), a.shape).cpu().numpy()
    if grid:
        np.testing.assert_array_equal(y, R.fwd_restate(a, c, w, b, fp, n_aggr))
        np.testing.assert_array_equal(ga, R.bwd_restate(gy, c, w, fp, n_aggr))
    else:
        want, bar = R.fwd_restate(a, c, w, b, fp, n_aggr, bars=True)
        assert (np.abs(y.astype(np.float64) - want) <= bar).all()
        want, bar = R.bwd_restate(gy, c, w, fp, n_aggr, bars=True)
        assert (np.abs(ga.astype(np.float64) - want) <= bar).all()


def test_autograd_matches_the_materialised_linear():
    """post_linear_towers_scaled against cat + baddbmm on the scaled copies: output and the gradients of a, weight, bias."""
    from pna_b200.linear import post_linear_towers_scaled
    n, t_n, fp, o, n_aggr, s_n = (1000, 5, 16, 14, 4, 3)
    a, c, w, b, gy = R.case_data((n, t_n, fp, o, n_aggr, s_n), grid=False)
    a1, w1, b1 = [_t(v).requires_grad_(True) for v in (a, w, b)]
    a2, w2, b2 = [_t(v).requires_grad_(True) for v in (a, w, b)]
    cs = _t(c)
    y1 = post_linear_towers_scaled(a1, cs, w1, b1)
    per = (1 + n_aggr) * fp
    at = a2.view(n, t_n, per)
    big = torch.cat([at[:, :, :fp]] + [at[:, :, fp:] * cs[:, s, None, None] for s in range(s_n)], dim=2)
    y2 = torch.baddbmm(b2.unsqueeze(1), big.transpose(0, 1), w2.transpose(1, 2)).transpose(0, 1).reshape(n, t_n * o)
    torch.testing.assert_close(y1, y2, rtol=1e-5, atol=1e-5)
    g = _t(gy)
    (y1 * g).sum().backward()
    (y2 * g).sum().backward()
    for p1, p2 in ((a1, a2), (w1, w2), (b1, b2)):
        torch.testing.assert_close(p1.grad, p2.grad, rtol=1e-4, atol=1e-4)


# ---- the layers --------------------------------------------------------------------------------------------------------
def _graph(n=2000, e=12000, seed=0):
    g = torch.Generator().manual_seed(seed)
    src, dst = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    dst[:50] = 7                                                   # a hub; rows that receive nothing are in-degree 0
    return src, dst, n


def _spy(monkeypatch):
    """Count the layers' calls of the tower kernel path; the small test graphs take it too (row threshold set to 0)."""
    from pna_b200 import dgl_layers, linear, pyg
    monkeypatch.setattr(linear, "TOWERS_COMPACT_MIN_ROWS", 0)
    calls = []
    real = pyg.post_linear_towers_scaled

    def spy(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(pyg, "post_linear_towers_scaled", spy)
    monkeypatch.setattr(dgl_layers, "post_linear_towers_scaled", spy)
    return calls


def _run(call, inputs, params):
    ins = [None if t is None else t.clone().requires_grad_(True) for t in inputs]
    out = call(*ins)
    w = torch.linspace(-1, 1, out.numel(), device=dev()).view_as(out)
    for p in params:
        p.grad = None
    (out * w).sum().backward()
    return out.detach(), [t.grad for t in ins if t is not None], [p.grad.clone() for p in params]


def _compare(make, monkeypatch):
    calls = _spy(monkeypatch)
    call, inputs, params = make()
    o1, gi1, gp1 = _run(call, inputs, params)
    assert calls, "compact tower path not taken"
    calls.clear()
    monkeypatch.setenv("PNA_B200_COMPACT_POST", "0")
    o2, gi2, gp2 = _run(call, inputs, params)
    monkeypatch.delenv("PNA_B200_COMPACT_POST")
    assert not calls
    torch.testing.assert_close(o1, o2, rtol=1e-5, atol=1e-5)
    for a, b in zip(gi1, gi2):                                   # input gradients: the golden tests' elementwise bar
        torch.testing.assert_close(a, b, rtol=1e-3, atol=5e-4)
    for a, b in zip(gp1, gp2):
        # parameter gradients sum over every row, with cancellation: the golden tests' bar, relative in the norm
        assert float((a - b).double().norm() / b.double().norm().clamp(min=1e-6)) < 2e-3


PYG = [dict(towers=4, divide_input=True), dict(towers=4, divide_input=False, fin=32), dict(towers=5, edge_dim=6, divide_input=True,
       fin=75, fout=75), dict(towers=2, pre_layers=2, post_layers=2), dict(towers=1, post_layers=2, fin=48, fout=48)]


@pytest.mark.parametrize("kw", PYG, ids=[str(i) for i in range(len(PYG))])
def test_pyg_conv_compact_path_matches_the_materialised_path(kw, monkeypatch):
    import pna_b200
    from pna_b200 import edge_mlp
    monkeypatch.setattr(edge_mlp, "FUSED_TRAINING_MIN_EDGES", 0)
    kw = dict(kw)
    fin, fout = kw.pop("fin", 64), kw.pop("fout", 64)

    def make():
        src, dst, n = _graph()
        ei = torch.stack([src, dst]).to(dev())
        deg = torch.bincount(torch.bincount(dst, minlength=n))
        torch.manual_seed(1)
        conv = pna_b200.PNAConv(fin, fout, ["mean", "min", "max", "std"], ["identity", "amplification", "attenuation"], deg,
                                **kw).to(dev())
        x = torch.randn(n, fin, device=dev())
        ea = torch.randn(src.numel(), kw["edge_dim"], device=dev()) if "edge_dim" in kw else None
        return (lambda x, ea: conv(x, ei, ea)), [x, ea], list(conv.parameters())
    _compare(make, monkeypatch)


DGL = [dict(towers=5, divide_input=True), dict(towers=5, divide_input=False, fin=16), dict(towers=5, edge_features=True, edge_dim=8),
       dict(towers=2, pretrans_layers=2, posttrans_layers=2, fin=32, fout=32)]


@pytest.mark.parametrize("kw", DGL, ids=[str(i) for i in range(len(DGL))])
def test_dgl_layer_compact_path_matches_the_materialised_path(kw, monkeypatch):
    import pna_b200
    from pna_b200 import edge_mlp
    monkeypatch.setattr(edge_mlp, "FUSED_TRAINING_MIN_EDGES", 0)
    kw = dict(kw)
    fin, fout = kw.pop("fin", 70), kw.pop("fout", 70)

    def make():
        src, dst, n = _graph()
        torch.manual_seed(2)
        lay = pna_b200.PNALayer(fin, fout, "mean max min std", "identity amplification attenuation", {"log": 1.6, "lin": 6.0},
                                0.0, True, True, **kw).to(dev())
        # the mixing network's LeakyReLU after the towers: a pre-activation within 1e-7 of 0 may take the other slope on
        # the other path and move a bias gradient by ~1e-1; the comparison is about the towers
        lay.mixing_network.activation = None
        graph = pna_b200.Graph(src, dst, n).to(dev())
        snorm = torch.rand(n, 1, device=dev())
        h = torch.randn(n, fin, device=dev())
        e = torch.randn(src.numel(), kw["edge_dim"], device=dev()) if kw.get("edge_features") else None
        return (lambda h, e: lay(graph, h, e, snorm)), [h, e], list(lay.parameters())
    _compare(make, monkeypatch)


def test_refused_shapes_keep_the_materialised_path(monkeypatch):
    """Shapes and dtypes the kernel does not take, and, at the default row threshold, small graphs and inference."""
    import pna_b200
    from pna_b200 import linear
    calls = _spy(monkeypatch)
    src, dst, n = _graph()
    ei = torch.stack([src, dst]).to(dev())
    deg = torch.bincount(torch.bincount(dst, minlength=n))
    x = torch.randn(n, 72, device=dev())
    for conv in (pna_b200.PNAConv(72, 72, ["mean", "max"], ["identity", "amplification"], deg, towers=1),      # O_t = 72
                 pna_b200.PNAConv(72, 72, ["mean", "max"], ["identity"], deg, towers=4),                        # S = 1
                 pna_b200.PNAConv(72, 72, ["mean", "max"], ["identity", "attenuation"], deg, towers=9, divide_input=True)):
        out = conv.to(dev())(x.requires_grad_(True), ei)
        out.sum().backward()
        assert torch.isfinite(out).all()
    lay = pna_b200.PNALayer(16, 16, "mean max", "identity amplification", {"log": 1.6}, 0.0, False, False,
                            towers=2).to(dev()).to(torch.bfloat16)
    out = lay(pna_b200.Graph(src, dst, n).to(dev()), torch.randn(n, 16, device=dev(), dtype=torch.bfloat16), None, None)
    assert out.dtype == torch.bfloat16
    monkeypatch.setattr(linear, "TOWERS_COMPACT_MIN_ROWS", 100_000)
    conv = pna_b200.PNAConv(72, 72, ["mean", "max"], ["identity", "amplification"], deg, towers=4, divide_input=True,
                            edge_dim=3).to(dev())
    ea = torch.randn(src.numel(), 3, device=dev())
    conv(x, ei, ea).sum().backward()                                     # 2000 rows: below TOWERS_COMPACT_MIN_ROWS
    monkeypatch.setattr(linear, "TOWERS_COMPACT_MIN_ROWS", 0)
    with torch.no_grad():
        conv(x, ei, ea)                                                  # inference
    assert not calls


def test_deterministic_training_steps_repeat_bit_for_bit(monkeypatch):
    import pna_b200
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    calls = _spy(monkeypatch)
    src, dst, n = _graph(seed=5)
    ei = torch.stack([src, dst]).to(dev())
    deg = torch.bincount(torch.bincount(dst, minlength=n))
    torch.manual_seed(3)
    dgl = pna_b200.PNALayer(70, 70, "mean max min std", "identity amplification attenuation", {"log": 1.6, "lin": 6.0}, 0.0, True,
                            True, towers=5).to(dev())
    conv = pna_b200.PNAConv(70, 70, ["mean", "min", "max", "std"], ["identity", "amplification", "attenuation"], deg, towers=5,
                            divide_input=True, post_layers=2).to(dev())
    graph = pna_b200.Graph(src, dst, n).to(dev())
    snorm = torch.full((n, 1), n ** -0.5, device=dev())
    h = torch.randn(n, 70, device=dev())
    models = torch.nn.ModuleList([dgl, conv])
    opt = torch.optim.SGD(models.parameters(), lr=1e-2)

    def two_steps():
        state = {k: v.clone() for k, v in models.state_dict().items()}
        grads = []
        for _ in range(2):
            x = h.clone().requires_grad_(True)
            opt.zero_grad()
            (dgl(graph, x, None, snorm).pow(2).mean() + conv(x, ei).pow(2).mean()).backward()
            grads.append([x.grad.clone()] + [p.grad.clone() for p in models.parameters()])
            opt.step()
        models.load_state_dict(state)
        return grads

    torch.use_deterministic_algorithms(True)
    try:
        g1, g2 = two_steps(), two_steps()
    finally:
        torch.use_deterministic_algorithms(False)
    assert calls
    for s1, s2 in zip(g1, g2):
        for a, b in zip(s1, s2):
            assert torch.equal(a, b)


def test_zinc_shaped_training_step_needs_less_memory(monkeypatch):
    """DGL PNALayer(70, 70, towers 5, divide_input) on a ZINC-shaped batch: the compact path's peak memory of a training step
    is below the materialised path's by at least the size of the [N, T (1 + S A) Fp] tensor it no longer writes."""
    import pna_b200
    from pna_b200 import linear, synth
    monkeypatch.setattr(linear, "TOWERS_COMPACT_MIN_ROWS", 0)
    ei, x, _ = synth.zinc_like(n_graphs=2000, n_feat=70)
    n = x.size(0)
    torch.manual_seed(0)
    lay = pna_b200.PNALayer(70, 70, "mean max min std", "identity amplification attenuation", {"log": 1.6, "lin": 2.2}, 0.0, True,
                            True, towers=5, divide_input=True).to(dev())
    graph = pna_b200.Graph(ei[0], ei[1], n).to(dev())
    snorm = torch.ones(n, 1, device=dev())
    h = x.to(dev())

    def peak():
        lay.zero_grad()
        hh = h.clone().requires_grad_(True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        lay(graph, hh, None, snorm).square().mean().backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    peak()                                                       # CSR, row scales: built once per graph
    compact = peak()
    monkeypatch.setenv("PNA_B200_COMPACT_POST", "0")
    peak()
    full = peak()
    materialised = n * 5 * (1 + 3 * 4) * 16 * 4
    assert full - compact >= materialised, (full, compact, materialised)
