"""Mixed precision on the H100: the bf16 kernel contracts bit for bit, and the tower layers, the dense layer and the readouts
trained under torch.autocast("cuda") in bf16 and fp16 (DESIGN section 2).

Bar for a layer: for its output and every gradient, the distance from the fp32 result without autocast is within 2.5x
that of the same module under the same autocast with the new kernels switched off (the torch message path and the
materialised tower path; for the dense layer, the fp32 edge-MLP kernel on widened operands), plus 1e-6 of the norm.
Parameter gradients are fp32."""
import contextlib

import pytest
import torch

import pna_b200
from pna_b200 import dense, edge_mlp, linear, readout, synth

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA GPU")]

A4 = ["mean", "max", "min", "std"]
S3 = ["identity", "amplification", "attenuation"]
DEV = "cuda"
AMP = {"bf16": torch.bfloat16, "fp16": torch.float16}


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32)


# ---- kernel contracts ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L,T,F,P,term", [(1, 5, 14, 16, True), (1, 1, 75, 80, True), (2, 5, 14, 16, True), (2, 4, 32, 32, False),
                                          (3, 2, 64, 64, True), (4, 5, 5, 8, False)])
def test_edge_messages_bf16_is_the_fp32_kernel_rounded_once(L, T, F, P, term):
    g = torch.Generator(device=DEV).manual_seed(L * 100 + F)
    n, e = 5000, 60_000
    ei = torch.randint(0, n, (2, e), device=DEV, generator=g)
    csr = pna_b200.csr_from_edge_index(ei, n)
    rnd = lambda *s: torch.randn(*s, device=DEV, generator=g)
    A, Bm = rnd(n, T * F).bfloat16(), rnd(n, T * F).bfloat16()
    C = rnd(e, T * F).bfloat16() if term else None
    b1 = 0.3 * rnd(T * F)
    W, bW = (rnd(L - 1, T, F, F) / F ** 0.5, 0.3 * rnd(L - 1, T, F)) if L > 1 else (b1.new_empty(0), b1.new_empty(0))
    M16, act16 = edge_mlp.edge_messages_forward(A, Bm, b1, W, bW, csr, T, C, P, store_activations=True)
    M32, act32 = edge_mlp.edge_messages_forward(A.float(), Bm.float(), b1, W, bW, csr, T, None if C is None else C.float(), P,
                                                store_activations=True)
    assert M16.dtype == torch.bfloat16 and torch.equal(_bits(M16), _bits(M32.bfloat16()))
    if L == 1:
        return
    assert act16.dtype == torch.bfloat16 and torch.equal(_bits(act16), _bits(act32.bfloat16()))
    dM = rnd(e, T * P).bfloat16()
    G16 = edge_mlp.edge_messages_backward(dM, P, act16, W, L, T, F)
    G32 = edge_mlp.edge_messages_backward(dM.float(), P, act16.float(), W, L, T, F)
    assert G16.dtype == torch.float32 and torch.equal(_bits(G16), _bits(G32))


@pytest.mark.parametrize("T,Fp,n_aggr,O,S", [(5, 16, 4, 14, 3), (4, 32, 4, 32, 3), (1, 64, 2, 64, 2), (8, 8, 6, 32, 5)])
def test_towers_bf16_is_the_fp32_kernel_on_the_widened_aggregate(T, Fp, n_aggr, O, S):
    g = torch.Generator(device=DEV).manual_seed(T * 10 + Fp)
    n = 1000 + 37                                               # a partial row tile
    a = torch.randn(n, T * (1 + n_aggr) * Fp, device=DEV, generator=g).bfloat16()
    rs = torch.rand(n, S, device=DEV, generator=g) * 2
    w = torch.randn(T, O, (1 + S * n_aggr) * Fp, device=DEV, generator=g) / 16
    b = torch.randn(T, O, device=DEV, generator=g)
    y16 = linear.linear_towers_scaled_tf32x3(a, rs, w, b)
    y32 = linear.linear_towers_scaled_tf32x3(a.float(), rs, w, b)
    assert y16.dtype == torch.float32 and torch.equal(_bits(y16), _bits(y32))


# ---- layers ------------------------------------------------------------------------------------------------------------
def _pyg(pre_layers=1, edge_dim=16, n_nodes=20_000, n_edges=200_000, width=64):
    ei, x = synth.arxiv_like(n_nodes=n_nodes, n_edges=n_edges, n_feat=width)
    deg = synth.degree_histogram(ei[1], n_nodes)
    torch.manual_seed(0)
    conv = pna_b200.PNAConv(width, width, A4, S3, deg, towers=4, divide_input=True, edge_dim=edge_dim, pre_layers=pre_layers).to(DEV)
    eid = ei.to(DEV)
    csr = pna_b200.csr_from_edge_index(eid, n_nodes)
    ea = torch.randn(n_edges, edge_dim, generator=torch.Generator().manual_seed(1)).to(DEV) if edge_dim else None
    return conv, (lambda xx: conv(xx, eid, ea, csr=csr)), x.to(DEV)


def _dgl(n_graphs=6000):
    ei, x, _ = synth.zinc_like(n_graphs=n_graphs, n_feat=70)
    n = x.size(0)
    e = torch.randn(ei.size(1), 50, generator=torch.Generator().manual_seed(1)).to(DEV)
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    torch.manual_seed(0)
    lay = pna_b200.PNALayer(70, 70, A4, S3, avg, 0.0, True, True, towers=5, divide_input=True, residual=True,
                            edge_features=True, edge_dim=50).to(DEV)
    graph = pna_b200.Graph(ei[0], ei[1], n).to(DEV)
    snorm = torch.ones(n, 1, device=DEV)
    return lay, (lambda hh: lay(graph, hh, e, snorm)), x.to(DEV)


def _dense():
    B, N, Fin = 8, 48, 32
    g = torch.Generator().manual_seed(3)
    adj = (torch.rand(B, N, N, generator=g) < 0.2).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float().to(DEV)
    x = torch.randn(B, N, Fin, generator=g).to(DEV)
    torch.manual_seed(0)
    lay = dense.PNALayer(Fin, Fin, A4, S3, {"log": 2.0, "lin": 9.6}, towers=2, pretrans_layers=2, divide_input=True).to(DEV)
    return lay, (lambda xx: lay(xx, adj)), x


def _step(mod, call, x, amp, seed=7):
    """Output and gradients (x and every parameter) of one forward + backward of a fixed random projection of the output."""
    mod.zero_grad(set_to_none=True)
    xg = x.clone().requires_grad_(True)
    ctx = torch.autocast("cuda", dtype=amp) if amp is not None else contextlib.nullcontext()
    with ctx:
        out = call(xg)
    r = torch.randn(out.shape, generator=torch.Generator(device=DEV).manual_seed(seed), device=DEV)
    (out.float() * r).sum().backward()
    res = {"out": out.detach().float(), "x": xg.grad.float()}
    for name, p in mod.named_parameters():
        if p.grad is not None:
            assert p.grad.dtype == torch.float32, name
            res[name] = p.grad.clone()
    assert xg.grad.dtype == x.dtype
    return res


def _check_bar(ref, new, off):
    assert set(new) == set(ref) == set(off)
    for k in ref:
        nrm = float(ref[k].double().norm())
        d_new = float((new[k].double() - ref[k].double()).norm())
        d_off = float((off[k].double() - ref[k].double()).norm())
        assert d_new <= 2.5 * d_off + 1e-6 * nrm, (k, d_new, d_off, nrm)


class _Spy:
    """Records the dtype of the operands the new kernel paths receive."""

    def __init__(self, monkeypatch):
        self.msgs, self.towers = [], []
        fwd, twr = edge_mlp.edge_messages_forward, linear.linear_towers_scaled_tf32x3
        monkeypatch.setattr(edge_mlp, "edge_messages_forward", lambda A, *a, **k: self.msgs.append(A.dtype) or fwd(A, *a, **k))
        monkeypatch.setattr(linear, "linear_towers_scaled_tf32x3", lambda a, *r, **k: self.towers.append(a.dtype) or twr(a, *r, **k))


def _off(monkeypatch):
    """The new kernel paths switched off: the torch message path in training, the materialised tower path."""
    monkeypatch.setattr(edge_mlp, "FUSED_TRAINING_MIN_EDGES", 1 << 62)
    monkeypatch.setenv("PNA_B200_COMPACT_POST", "0")


CASES = {
    "pyg_edges_L1": (lambda: _pyg(pre_layers=1), True, False),     # (make, fused messages, compact towers)
    "pyg_edges_L2": (lambda: _pyg(pre_layers=2), True, False),
    "pyg_compact": (lambda: _pyg(edge_dim=None, n_nodes=110_000, n_edges=600_000, width=128), False, True),
    "dgl_zinc_edges_compact": (lambda: _dgl(), True, True),
}


@pytest.mark.parametrize("amp", list(AMP))
@pytest.mark.parametrize("case", list(CASES))
def test_tower_layers_under_autocast(case, amp, monkeypatch):
    make, fused, compact = CASES[case]
    mod, call, x = make()
    n = x.size(0)
    assert (n >= linear.TOWERS_COMPACT_MIN_ROWS) == compact
    ref = _step(mod, call, x, None)
    spy = _Spy(monkeypatch)
    new = _step(mod, call, x, AMP[amp])
    want = torch.bfloat16 if amp == "bf16" else torch.float32
    assert spy.msgs == ([want] if fused else []) and spy.towers == ([want] if compact else [])
    with monkeypatch.context() as m:
        _off(m)
        spy.msgs.clear(), spy.towers.clear()
        off = _step(mod, call, x, AMP[amp])
        assert spy.msgs == [] and spy.towers == []
    _check_bar(ref, new, off)
    # layer 2 onward of a real net: a bf16 input takes the same kernels
    spy.msgs.clear(), spy.towers.clear()
    if amp == "bf16":
        with torch.autocast("cuda", dtype=torch.bfloat16):
            call(x.bfloat16().requires_grad_(True)).float().sum().backward()
        assert spy.msgs == ([torch.bfloat16] if fused else []) and spy.towers == ([torch.bfloat16] if compact else [])


def test_compact_path_saves_a_bf16_aggregate():
    mod, call, x = _pyg(edge_dim=None, n_nodes=110_000, n_edges=600_000, width=128)
    saved = []

    def pack(t):
        saved.append((t.dtype, tuple(t.shape)))
        return t

    width = 4 * (1 + len(A4)) * 32                        # T * (1 + A) * Fp
    with torch.autograd.graph.saved_tensors_hooks(pack, lambda t: t):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = call(x.clone().requires_grad_(True))
    out.float().sum().backward()
    assert (torch.bfloat16, (x.size(0), width)) in saved
    assert (torch.float32, (x.size(0), width)) not in saved


@pytest.mark.parametrize("amp", list(AMP))
def test_dense_layer_with_two_pretrans_layers_under_autocast(amp, monkeypatch):
    mod, call, x = _dense()
    ref = _step(mod, call, x, None)
    spy = _Spy(monkeypatch)
    new = _step(mod, call, x, AMP[amp])
    assert spy.msgs == ([torch.bfloat16] if amp == "bf16" else [])
    with monkeypatch.context() as m:
        m.setattr(dense, "at_boundary", lambda t: t.float())      # the fp32 edge-MLP kernel on widened operands
        off = _step(mod, call, x, AMP[amp])
    _check_bar(ref, new, off)


@pytest.mark.parametrize("amp", list(AMP))
def test_readouts_under_autocast(amp):
    """An autocast Linear's output through every readout: fp16 is reduced in fp32 (the fp32 readout of the widened input,
    bit for bit); bf16 stays bf16, the fp32 readout of the widened input rounded once."""
    n, g = 5000, 37
    batch = torch.sort(torch.randint(0, g, (n,), generator=torch.Generator().manual_seed(0)))[0].to(DEV)
    lin = torch.nn.Linear(16, 24).to(DEV)
    x0 = torch.randn(n, 16, device=DEV)
    for fn in (readout.global_add_pool, readout.global_mean_pool, readout.global_max_pool):
        xg = x0.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=AMP[amp]):
            h = lin(xg)
            y = fn(h, batch, g)
        assert h.dtype == AMP[amp]
        want = fn(h.detach().float(), batch, g)
        if amp == "fp16":
            assert y.dtype == torch.float32 and torch.equal(y, want)
        else:
            assert y.dtype == torch.bfloat16 and torch.allclose(y.float(), want, rtol=2 ** -8, atol=0)
        y.float().sum().backward()
        assert xg.grad is not None and xg.grad.dtype == torch.float32 and torch.isfinite(xg.grad).all()
