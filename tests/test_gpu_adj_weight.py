"""Slot weights on the H100: the aggregation with slot weights / a real scaler degree (pna_aggregate_*_weighted) against the unweighted kernels
(all-ones and power-of-two weights), against float64 within the bars of tests/adj_weight_bars.py (random and signed weights,
split rows included), and the dense PNALayer on a weighted adjacency against the reference's own layer
(tests/golden/dense_adj_weighted.pt), deterministic, captured and under autocast."""
import math
import os

import pytest
import torch

import adj_weight_bars as AB
from pna_b200 import aggregate as agg, csr_from_edge_index, dense
from test_gpu_capture import _mode, _replay_matches_eager

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
SIX = ["mean", "max", "min", "std", "sum", "var"]
AVG = {"log": 1.7, "lin": 4.5}
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "dense_adj_weighted.pt")


def graph(n, e, seed, hub=0):
    """Random multigraph on n nodes; `hub` extra in-edges of node 0 (a split row when above the split threshold)."""
    g = torch.Generator().manual_seed(seed)
    src, dst = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    if hub:
        src = torch.cat([src, torch.randint(0, n, (hub,), generator=g)])
        dst = torch.cat([dst, torch.zeros(hub, dtype=torch.long)])
    ei = torch.stack([src, dst]).to(DEV)
    return ei, csr_from_edge_index(ei, n), g


def slot_weights(csr, kind, g):
    E = csr.n_edges
    if kind == "ones":
        w = torch.ones(E)
    elif kind in ("two", "half"):
        w = torch.full((E,), 2.0 if kind == "two" else 0.5)
    else:
        w = torch.rand(E, generator=g) * 1.75 + 0.25
        if kind == "signed":
            neg = torch.rand(E, generator=g) < 0.1
            w[neg] = -0.25 * torch.rand(int(neg.sum()), generator=g) - 0.05
    return w.to(DEV).contiguous()


def light(csr):
    return (csr.in_degree < csr.split_threshold).cpu()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_all_ones_and_power_of_two_weights_reproduce_the_unweighted_kernel(dtype):
    ei, csr, g = graph(3000, 24000, 1)
    x = (torch.randn(3000, 64, generator=g) * 2).to(DEV, dtype)
    scal = ["identity", "amplification", "attenuation"]
    ref = agg.aggregate_forward(x, csr, SIX, scal, AVG, relu_var=True).cpu()
    lt = light(csr)
    assert lt.all()
    ones = agg.aggregate_forward(x, csr, SIX, scal, AVG, relu_var=True, slot_weight=slot_weights(csr, "ones", g)).cpu()
    assert torch.equal(ones[lt], ref[lt])
    F = 64
    for kind, k in (("two", 2.0), ("half", 0.5)):
        out = agg.aggregate_forward(x, csr, SIX, scal, AVG, relu_var=True, slot_weight=slot_weights(csr, kind, g)).cpu()
        for s in range(3):
            for a, name in enumerate(SIX):
                cols = slice((s * 6 + a) * F, (s * 6 + a + 1) * F)
                want = ref[:, cols] * k if name == "sum" else ref[:, cols]
                assert torch.equal(out[lt][:, cols], want[lt].to(dtype) if dtype == torch.bfloat16 else want[lt]), (kind, name)


def test_all_ones_deterministic_backward_reproduces_the_unweighted_bits():
    ei, csr, g = graph(2000, 16000, 2)
    x = torch.randn(2000, 32, generator=g).to(DEV)
    bias = torch.randn(2000, 32, generator=g).to(DEV)
    go = torch.randn(2000, 6 * 2 * 32, generator=g).to(DEV)
    kw = dict(row_bias=bias, need_bias_grad=True, relu_var=True)
    with _mode(True):
        want = agg.aggregate_backward(go, x, csr, SIX, ["identity", "linear"], AVG, **kw)
        got = agg.aggregate_backward(go, x, csr, SIX, ["identity", "linear"], AVG, slot_weight=slot_weights(csr, "ones", g), **kw)
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])


def _slot_order(csr, ei):
    """edge ids of the CSR slots and the destination of every edge"""
    return csr.perm.long().cpu(), ei[1].cpu()


@pytest.mark.parametrize("kind", ["pos", "signed"])
@pytest.mark.parametrize("hub", [0, 5000])
def test_random_weights_within_the_bar_forward_and_slot_gradients(kind, hub):
    n = 1500
    ei, csr, g = graph(n, 9000, 3 + hub, hub=hub)
    if hub:
        assert csr.n_hubs >= 1
    F = 32
    x = (torch.randn(n, F, generator=g) + 0.5).to(DEV)
    w = slot_weights(csr, kind, g)
    perm, dst = _slot_order(csr, ei)
    w_edge = torch.empty_like(w.cpu())
    w_edge[perm] = w.cpu()
    msg = x.cpu()[ei[0].cpu()]
    out = agg.aggregate_forward(x, csr, SIX, ["identity", "attenuation"], AVG, relu_var=True, slot_weight=w).cpu()
    ref = AB.forward(msg, w_edge, dst, n)
    D = csr.in_degree.double().cpu()
    att = torch.where(D > 0, AVG["log"] / torch.log(D + 1), torch.ones_like(D)).unsqueeze(1)
    for a, name in enumerate(SIX):
        y, bar = ref[name]
        got = out[:, a * F:(a + 1) * F].double()
        assert ((got - y).abs() <= bar).all(), (name, float(((got - y).abs() - bar).max()))
        ys, bs = AB.scaled_bar(y, bar, att)
        gs = out[:, (6 + a) * F:(7 + a) * F].double()
        assert ((gs - ys).abs() <= bs).all(), (name, "attenuation")
    # per-slot gradients: messages in CSR order, so the backward's result IS the slot gradient (both modes)
    m_csr = x[ei[0][csr.perm.long()]].contiguous()
    go = torch.randn(n, 6 * F, generator=g).to(DEV)
    G = {name: go.cpu()[:, a * F:(a + 1) * F] for a, name in enumerate(SIX)}
    want, bar = AB.slot_grads(msg, w_edge, dst, n, G)
    for det in (True, False):
        with _mode(det):
            gs, _ = agg.aggregate_backward(go, m_csr, csr, SIX, ["identity"], AVG, messages_in_csr_order=True, relu_var=True,
                                           slot_weight=w)
        err = (gs.cpu().double() - want[perm]).abs()
        assert (err <= bar[perm]).all(), (det, float((err - bar[perm]).max()))


# ---- the dense layer ---------------------------------------------------------------------------------------------------
def _golden():
    return torch.load(GOLDEN, weights_only=False)


@pytest.mark.parametrize("key", ["False_1_True", "False_1_False", "True_1_True", "True_1_False", "False_2_True",
                                 "False_2_False", "True_2_True", "True_2_False", "negD_1", "negD_2"])
def test_golden_dense_layer_on_a_weighted_adjacency(key):
    """negD_*: identity / mean / max / std on an adjacency with a row sum D in (-1, 0), where attenuation and inverse_linear
    divide by log(D + 1) < 0 and D < 0 (1 only where D == 0), in the kernels and in the identity block alike."""
    g = _golden()
    c = g["cases"][key]
    lay = dense.PNALayer(aggregators=c["aggregators"], scalers=g["scalers"], avg_d=c["avg_d"], **c["ctor"])
    lay.load_state_dict(c["state_dict"])
    lay = lay.to(DEV).eval()
    adj = c["adj"].to(DEV)
    if key.startswith("negD"):
        D = adj.sum(-1)
        assert bool(((D > -1) & (D < 0)).any())
    graphs = dense.dense_graphs(adj, c["ctor"]["self_loop"])
    assert graphs.row_weight is not None and graphs.scaler_degree.dtype == torch.float32
    with torch.no_grad():
        out = lay(g["h"].to(DEV), adj).cpu()
    ref64, ref32 = c["out64"], c["out"]
    err = (out.double() - ref64).abs()
    lim = torch.maximum(1e-5 + 1e-5 * ref64.abs(), 2.5 * (ref32.double() - ref64).abs())
    assert (err <= lim).all(), float((err / lim).max())
    h = g["h"].to(DEV).requires_grad_(True)
    (lay(h, adj) * c["grads"]["w"].to(DEV)).sum().backward()
    torch.testing.assert_close(h.grad.cpu(), c["grads"]["h"], rtol=1e-3, atol=5e-4)
    # and relative to its norm, as the parameter gradients: the input gradients are 1e-4..1e-3, near the atol above
    ref = c["grads"]["h"]
    assert float((h.grad.cpu() - ref).norm() / ref.norm()) < 2e-3
    for k, p in lay.named_parameters():
        ref = c["grads"]["params"][k]
        rel = float((p.grad.cpu() - ref).norm() / ref.norm().clamp(min=1e-6))
        assert rel < 2e-3, f"{k}: {rel:.2e}"


def _weighted_case(pretrans_layers=1, self_loop=False, B=64, N=32, F=16):
    """A weighted adjacency: entries in [0.25, 2], about 10 % of them negative and small (at most 0.2 in magnitude), and one
    entry of 1.5 in every row, so that no row's weights nearly cancel (W_i >= 0.5 on these shapes)."""
    gen = torch.Generator().manual_seed(5)
    mask = (torch.rand(B, N, N, generator=gen) < 0.2).float() * (1 - torch.eye(N))
    w = torch.rand(B, N, N, generator=gen) * 1.75 + 0.25
    w = torch.where(torch.rand(B, N, N, generator=gen) < 0.1, -0.1 * w, w)
    adj = mask * w
    adj[:, torch.arange(N), (torch.arange(N) + 1) % N] = 1.5
    assert float(adj.sum(-1).min()) >= 0.5
    adj = adj.to(DEV)
    torch.manual_seed(0)
    m = dense.PNALayer(F, F, SIX, ["identity", "amplification", "attenuation"], {"log": 1.6, "lin": 4.8}, towers=2,
                       pretrans_layers=pretrans_layers, self_loop=self_loop, divide_input=True).to(DEV)
    return m, {"x": torch.randn(B, N, F, generator=gen).to(DEV)}, lambda m, i: m(i["x"], adj)


def _step(m, inputs, run):
    x = inputs["x"].detach().clone().requires_grad_(True)
    m.zero_grad()
    out = run(m, {"x": x})
    (out * torch.linspace(-1, 1, out.numel(), device=DEV).view(out.shape)).sum().backward()
    return [out.detach(), x.grad] + [p.grad.clone() for p in m.parameters()]


@pytest.mark.parametrize("pre", [1, 2])
def test_deterministic_training_step_repeats_and_matches_the_atomic_mode(pre):
    m, inputs, run = _weighted_case(pretrans_layers=pre)
    with _mode(True):
        a, b = _step(m, inputs, run), _step(m, inputs, run)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    with _mode(False):
        c = _step(m, inputs, run)
    for u, v in zip(a, c):
        assert float((u - v).abs().max()) <= 1e-4 * float(u.abs().max()) + 1e-6


@pytest.mark.parametrize("pre,self_loop", [(1, False), (2, True)])
@pytest.mark.parametrize("train", [False, True])
def test_captured_weighted_step_equals_the_eager_step(pre, self_loop, train):
    with _mode(True):
        m, inputs, run = _weighted_case(pretrans_layers=pre, self_loop=self_loop)
        _replay_matches_eager(m, inputs, run, train=train, exact=True)


def _torch_weighted_aggregate(gathered, csr, aggregators, scalers, avg_deg, *, towers=1, row_bias=None, self_feat=None,
                              self_divided=True, messages_in_csr_order=False, relu_var=False, scaler_degree=None,
                              slot_weight=None, out=None, **_):
    """The weighted aggregation restated in torch (fp32, autograd), same column layout: the yardstick of the autocast test."""
    N = csr.n_nodes
    g = gathered.float()
    m = g if messages_in_csr_order else g[csr.col.long()]
    dst = csr.dst_of_slot.long()
    if row_bias is not None:
        m = m + row_bias.float()[dst]
    F = m.size(1)
    w = slot_weight if slot_weight is not None else torch.ones(m.size(0), device=m.device)
    W = torch.zeros(N, device=m.device).index_add(0, dst, w).unsqueeze(1)
    S = torch.zeros(N, F, device=m.device).index_add(0, dst, m * w[:, None])
    Q = torch.zeros(N, F, device=m.device).index_add(0, dst, m * m * w[:, None])
    deg = csr.in_degree.unsqueeze(1)
    has = deg > 0
    mean = torch.where(has, S / W, 0.0)
    var = torch.where(has, Q / W - mean * mean, 0.0)
    pos = (w > 0)[:, None].expand_as(m)
    mx = torch.full((N, F), -math.inf, device=m.device).scatter_reduce(0, dst[:, None].expand_as(m), torch.where(pos, m, -math.inf), "amax")
    mn = torch.full((N, F), math.inf, device=m.device).scatter_reduce(0, dst[:, None].expand_as(m), torch.where(pos, m, math.inf), "amin")
    vals = dict(sum=S, mean=mean, var=var.clamp(min=0) if relu_var else var, std=(var.clamp(min=0) + 1e-5).sqrt(),
                max=torch.where(torch.isinf(mx), 0.0, mx), min=torch.where(torch.isinf(mn), 0.0, mn))
    D = (scaler_degree if scaler_degree is not None else csr.in_degree).float().unsqueeze(1)
    lg = torch.log(D + 1)
    fac = dict(identity=torch.ones_like(D), amplification=lg / avg_deg["log"],
               attenuation=torch.where(D != 0, avg_deg["log"] / lg, 1.0), linear=D / avg_deg.get("lin", 1.0),
               inverse_linear=torch.where(D != 0, avg_deg.get("lin", 1.0) / D, 1.0))
    Ft = F // towers
    blocks = []
    for t in range(towers):
        sl = slice(t * Ft, (t + 1) * Ft)
        parts = []
        if self_feat is not None:
            parts.append(self_feat.float()[:, sl] if self_divided else self_feat.float()[:, :Ft])
        for s in agg._names(scalers):
            for a in agg._names(aggregators):
                parts.append(torch.zeros(N, Ft, device=m.device) if a == "_skip" else vals[a][:, sl] * fac[s])
        blocks.append(torch.cat(parts, 1))
    res = torch.cat(blocks, 1).to(gathered.dtype)
    if out is None:
        return res
    # written columns only (PNA_AGGR_SKIP keeps the other call's): per tower the self block, then every non-skipped slot
    col = [True] * (Ft if self_feat is not None else 0)
    for s in agg._names(scalers):
        for a in agg._names(aggregators):
            col += [a != "_skip"] * Ft
    mask = torch.tensor(col * towers, device=m.device)
    out.copy_(torch.where(mask, res, out))          # in place, as the kernel writes into `out`
    return out


@pytest.mark.parametrize("pre", [1, 2])
@pytest.mark.parametrize("amp", [torch.bfloat16, torch.float16])
def test_autocast_distance_within_that_of_a_torch_restatement(amp, pre, monkeypatch):
    """pre = 1: the affine path (its messages Bm + b are fp32 under autocast); pre = 2: the edge-MLP path, whose bf16 messages
    reach the bf16 instances of the weighted kernels under bf16 autocast."""
    m, inputs, run = _weighted_case(pretrans_layers=pre)
    with torch.no_grad():
        y32 = run(m, inputs).float()
        with torch.autocast("cuda", dtype=amp):
            ya = run(m, inputs).float()
        monkeypatch.setattr(dense, "pna_aggregate", _torch_weighted_aggregate)
        monkeypatch.setattr(dense, "aggregate_forward", _torch_weighted_aggregate)
        t32 = run(m, inputs).float()
        with torch.autocast("cuda", dtype=amp):
            ta = run(m, inputs).float()
    assert float((t32 - y32).abs().max()) <= 1e-4 * float(y32.abs().max())     # the restatement computes the same layer
    d_kernel, d_torch = float((ya - y32).norm()), float((ta - t32).norm())
    assert d_kernel <= 2.5 * d_torch + 1e-6 * float(y32.norm()), (d_kernel, d_torch)


def test_refusals_raise_before_any_launch():
    adj = (torch.rand(4, 8, 8) * 2).to(DEV)
    for a in (["mean", "softmax"], ["moment3"], ["normalised_mean"]):
        lay = dense.PNALayer(8, 8, a, ["identity"], {"log": 1.0, "lin": 1.0}).to(DEV)
        with pytest.raises(NotImplementedError):
            lay(torch.randn(4, 8, 8, device=DEV), adj)
    lay = dense.PNALayer(8, 8, ["mean", "max"], ["identity"], {"log": 1.0, "lin": 1.0}).to(DEV)
    bad = adj.clone()
    bad[0, 1, 2] = float("nan")
    with pytest.raises(ValueError):
        lay(torch.randn(4, 8, 8, device=DEV), bad)
    leaf = adj.clone().requires_grad_(True)
    with pytest.raises(ValueError):
        lay(torch.randn(4, 8, 8, device=DEV), leaf)
    # what the message asks for then works: the cached graph of this adjacency holds no autograd history
    graphs = dense.dense_graphs(leaf.detach(), False)
    assert not graphs.row_weight.requires_grad and not graphs.scaler_degree.requires_grad
    assert torch.isfinite(lay(torch.randn(4, 8, 8, device=DEV), leaf.detach())).all()
    ei, csr, g = graph(100, 500, 9)
    x = torch.randn(100, 8, device=DEV)
    w = slot_weights(csr, "pos", g)
    with pytest.raises(NotImplementedError):
        agg.aggregate_forward(x, csr, ["mean", "moment4"], ["identity"], AVG, slot_weight=w)
    with pytest.raises(ValueError):
        agg.pna_aggregate(x.requires_grad_(True), csr, ["mean"], ["identity"], AVG, slot_weight=w.requires_grad_(True))
    torch.cuda.synchronize()


@pytest.mark.parametrize("pre", [1, 2])
def test_a_01_adjacency_keeps_the_unweighted_path(pre, monkeypatch):
    """A float 0/1 adjacency: int32 degree, no slot weights, and no call of the layer (forward and training) reaches the
    weighted entry points; the same pattern with real weights reaches them in every call of the layer's aggregators (the
    deterministic backward's unweighted "sum" over the reversed slots excepted)."""
    mask = ((torch.rand(8, 16, 16, generator=torch.Generator().manual_seed(2)) < 0.3).float() * (1 - torch.eye(16))).to(DEV)
    graphs = dense.DenseGraphs(mask)
    assert graphs.row_weight is None and graphs.scaler_degree.dtype == torch.int32
    seen = []
    real = agg._weights
    def spy(w, aggregators, *a, **k):
        r = real(w, aggregators, *a, **k)
        if list(aggregators) != ["sum"]:
            seen.append(r)
        return r
    monkeypatch.setattr(agg, "_weights", spy)
    lay = dense.PNALayer(16, 16, SIX, ["identity", "amplification"], {"log": 1.6, "lin": 4.8}, towers=2,
                         pretrans_layers=pre).to(DEV)
    x = torch.randn(8, 16, 16, device=DEV, requires_grad=True)
    lay(x, mask).sum().backward()
    assert seen and all(w is None for w in seen)
    seen.clear()
    lay(x, mask * 1.5).sum().backward()
    assert seen and all(w is not None for w in seen)
