"""The tensor-core linear's backward on the GPU (pna_linear_bwd_data / pna_linear_bwd_weight, 3xTF32 wgmma).

Accuracy is measured as in DESIGN section 2 for a dot product: elementwise |g - g64| / (sum of |products|), g64 the float64
gradient of what the forward multiplied (for the compact path: of the fp32 scaled copies fl(c_s * a)).  The bar is 1e-5 and
2.5x the error of the library fp32 GEMMs the backward used before (restated in `library_grads`) plus 1e-7.  A gradient
that is ONE product (dW with a single row) is held to 3 * 2^-22 instead: 3xTF32 carries each operand to 2^-22 relative
(the rounded lo part and the dropped lo.lo term) where fp32 carries it to 2^-24, and with one product no sum dilutes that."""
import pytest
import torch

pytestmark = pytest.mark.gpu

A4 = ["mean", "max", "min", "std"]
S3 = ["identity", "amplification", "attenuation"]
ONE_PRODUCT = 3 * 2.0 ** -22


def dev():
    return torch.device("cuda:0")


@pytest.fixture(autouse=True)
def _keep_global_rng():
    """The layer tests seed torch's global generators; restore them so that later modules draw what they would without
    this one."""
    with torch.random.fork_rng(devices=[torch.cuda.current_device()]):
        yield


@pytest.fixture(scope="module", autouse=True)
def _release_memory():
    """The long-chain cases allocate several GB; hand the cached blocks back to later modules."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def scaled_operand(a, c):
    """cat_s(fl32(c_s * a)): the operand the forward's loaders form (the plain operand when c is None)."""
    return a if c is None else torch.cat([a * c[:, s:s + 1] for s in range(c.size(1))], dim=1)


def exact_grads(gy, a, c, w):
    """float64 (ga, gw) of y = scaled_operand(a, c) @ w.T, and the sum of |products| of every element."""
    ka = a.size(1)
    s_n = 1 if c is None else c.size(1)
    gy64 = gy.double()
    a1 = scaled_operand(a, c).double()
    gw64, gw_cond = gy64.t() @ a1, gy64.abs().t() @ a1.abs()
    ga64 = torch.zeros(a.shape, dtype=torch.float64, device=a.device)
    ga_cond = torch.zeros_like(ga64)
    for s in range(s_n):
        ws = w[:, s * ka:(s + 1) * ka].double()
        cs = torch.ones((a.size(0), 1), dtype=torch.float64, device=a.device) if c is None else c[:, s:s + 1].double()
        ga64 += cs * (gy64 @ ws)
        ga_cond += cs.abs() * (gy64.abs() @ ws.abs())
    return (ga64, ga_cond), (gw64, gw_cond)


def library_grads(gy, a, c, w):
    """The library-GEMM backward this kernel pair replaced, verbatim (fp32, one scaler block at a time)."""
    if c is None:
        return gy @ w, gy.t() @ a
    ka = a.size(1)
    ga, gw = torch.zeros_like(a), torch.empty_like(w)
    for s in range(c.size(1)):
        cs = c[:, s:s + 1]
        ga.addcmul_(gy @ w[:, s * ka:(s + 1) * ka], cs)
        torch.mm(gy.t(), a * cs, out=gw[:, s * ka:(s + 1) * ka])
    return ga, gw


def rel_err(g, ref):
    g64, cond = ref
    d = (g.double() - g64).abs()
    return float(torch.where(cond > 0, d / cond.clamp(min=1e-300), d * float("inf")).nan_to_num(0.0).max())


def check_bound(name, got, lib, floor=0.0):
    assert got <= 1e-5 and got <= max(2.5 * lib + 1e-7, floor), f"{name}: {got:.3e} (library fp32: {lib:.3e})"


def make(n, ka, s, o, seed, zero_scale=True, device=None):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(n, ka, generator=g)
    c = None
    if s:
        c = torch.rand(n, s, generator=g) * 3
        c[:, 0] = 1.0
        if zero_scale and n > 5:
            c[5, 1] = 0.0                                           # amplification of an isolated row
    w = torch.randn(o, (s or 1) * ka, generator=g) / ((s or 1) * ka) ** 0.5
    gy = torch.randn(n, o, generator=g)
    d = device or dev()
    return gy.to(d), a.to(d), None if c is None else c.to(d), w.to(d)


def check_case(gy, a, c, w):
    from pna_b200 import linear as L
    ga, gw = L.linear_bwd_tf32x3(gy, a, c, w)
    torch.cuda.synchronize()
    (ga_ref, gw_ref) = exact_grads(gy, a, c, w)
    lga, lgw = library_grads(gy, a, c, w)
    check_bound("grad a", rel_err(ga, ga_ref), rel_err(lga, ga_ref))
    check_bound("grad weight", rel_err(gw, gw_ref), rel_err(lgw, gw_ref), ONE_PRODUCT if a.size(0) == 1 else 0.0)
    return ga, gw


@pytest.mark.parametrize("n,k,o", [(1, 32, 64), (127, 64, 128), (4097, 1536, 128), (300, 320, 256)])
def test_plain_backward_against_float64(n, k, o):
    check_case(*make(n, k, 0, o, seed=n + k + o))


@pytest.mark.parametrize("n,ka,s,o", [(1, 32, 3, 64), (129, 64, 2, 128), (4099, 512, 3, 128), (700, 96, 5, 256)])
def test_compact_backward_against_float64(n, ka, s, o):
    gy, a, c, w = make(n, ka, s, o, seed=n + ka + s + o)
    ga, gw = check_case(gy, a, c, w)
    if n > 5:                                                      # the zero factor: that copy contributes nothing to row 5
        ref = sum(c[5, i] * (gy[5:6].double() @ w[:, i * ka:(i + 1) * ka].double()) for i in range(s) if i != 1)
        assert float((ga[5:6].double() - ref).abs().max()) <= 1e-5 * float(ref.abs().max())


@pytest.mark.parametrize("n", [169_343, 1_000_003])
def test_long_accumulation_chain_weight_gradient(n):
    """dW reduces over all N rows.  The tensor core adds with truncation, a bias that grows with the chain; folding every 64
    rows into a round-to-nearest partial keeps it below the library's own rms error."""
    from pna_b200 import linear as L
    g = torch.Generator(device=dev()).manual_seed(n)
    ka, s, o = 512, 3, 128
    a = torch.randn(n, ka, generator=g, device=dev())
    c = torch.rand(n, s, generator=g, device=dev()) * 3
    c[:, 0] = 1.0
    gy = torch.randn(n, o, generator=g, device=dev())
    w = torch.randn(o, s * ka, generator=g, device=dev()) / (s * ka) ** 0.5
    _, gw = L.linear_bwd_tf32x3(gy, a, c, w, need_a=False)
    _, lgw = library_grads(gy, a, c, w)
    gy64 = gy.double()
    for i in range(s):                                              # float64 reference, one scaler block at a time
        cols = slice(i * ka, (i + 1) * ka)
        a1 = (a * c[:, i:i + 1]).double()
        ref = (gy64.t() @ a1, gy64.abs().t() @ a1.abs())
        del a1
        check_bound(f"grad weight block {i}", rel_err(gw[:, cols], ref), rel_err(lgw[:, cols], ref))
        d = gw[:, cols].double() - ref[0]
        bias = float((d * torch.sign(ref[0])).mean())               # < 0: results shrink towards zero
        rms_lib = float((lgw[:, cols].double() - ref[0]).pow(2).mean().sqrt())
        assert abs(bias) < rms_lib, f"block {i}: signed bias {bias:.3e} vs library rms error {rms_lib:.3e}"


def test_repeatable_strided_and_partial():
    from pna_b200 import linear as L
    gy, a, c, w = make(5003, 96, 3, 64, seed=7)                     # N a multiple of no tile or split
    ga1, gw1 = L.linear_bwd_tf32x3(gy, a, c, w)
    ga2, gw2 = L.linear_bwd_tf32x3(gy, a, c, w)
    assert torch.equal(ga1, ga2) and torch.equal(gw1, gw2)
    # a non-contiguous upstream gradient (every other column of a wider one) gives the same bits
    wide = torch.zeros(gy.size(0), 2 * gy.size(1), device=dev())
    wide[:, ::2] = gy
    ga3, gw3 = L.linear_bwd_tf32x3(wide[:, ::2], a, c, w)
    assert torch.equal(ga1, ga3) and torch.equal(gw1, gw3)
    # pitched a (a column slice of a wider tensor): what the layers' kernel_applies admits
    aw = torch.randn(a.size(0), 160, device=dev())
    aw[:, 32:128] = a
    ga4, gw4 = L.linear_bwd_tf32x3(gy, aw[:, 32:128], c, w)
    assert torch.equal(ga1, ga4) and torch.equal(gw1, gw4)
    only_a = L.linear_bwd_tf32x3(gy, a, c, w, need_w=False)
    only_w = L.linear_bwd_tf32x3(gy, a, c, w, need_a=False)
    assert only_a[1] is None and torch.equal(only_a[0], ga1)
    assert only_w[0] is None and torch.equal(only_w[1], gw1)


@pytest.mark.parametrize("scaled", [False, True])
def test_autograd_needs_input_grad(scaled):
    from pna_b200 import linear as L
    gy, a, c, w = make(777, 64, 3 if scaled else 0, 128, seed=3)
    b = torch.randn(128, device=dev())

    def run(a_grad, w_grad):
        a_ = a.clone().requires_grad_(a_grad)
        w_ = w.clone().requires_grad_(w_grad)
        b_ = b.clone().requires_grad_(True)
        y = L.post_linear_scaled(a_, c, w_, b_) if scaled else L.post_linear(a_, w_, b_)
        (y * gy).sum().backward()
        return a_.grad, w_.grad, b_.grad
    ga, gw, gb = run(True, True)
    want_a, _ = L.linear_bwd_tf32x3(gy, a, c, w, need_w=False)
    want_w = L.library_grad_weight(gy, a, c, w)                     # cuBLAS is faster than pna_linear_bwd_weight at config 2
    assert torch.equal(ga, want_a) and torch.equal(gw, want_w)
    torch.testing.assert_close(gb, gy.sum(0))
    ga, gw, gb = run(True, False)                                   # frozen weight: no weight gradient
    assert gw is None and torch.equal(ga, want_a)
    ga, gw, gb = run(False, True)                                   # constant input: no input gradient
    assert ga is None and torch.equal(gw, want_w)


@pytest.fixture
def deterministic(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


def _graph(n, e, seed):
    """Random graph without repeated edges (a repeated edge ties min / max, whose gradient routing is not at stake here)."""
    g = torch.Generator().manual_seed(seed)
    dst = torch.randint(0, int(n * 0.85), (e,), generator=g)
    src = torch.randint(0, n, (e,), generator=g)
    key = torch.unique(dst * n + src)
    return torch.stack([key % n, key // n])


def test_pnaconvsimple_gradients_match_oracle():
    """One post layer: with two, a ReLU between them whose input lies within rounding of zero may flip between the GPU and
    the CPU oracle and move whole rows of x.grad (the repeatability test below runs two layers)."""
    import pna_b200 as P
    from oracle import pna_oracle as O
    n, f = 3000, 64
    ei = _graph(n, 24000, 5)
    x = torch.randn(n, f, generator=torch.Generator().manual_seed(6))
    deg = torch.bincount(torch.bincount(ei[1], minlength=n))
    torch.manual_seed(0)
    ref = O.PNAConvSimpleOracle(f, 128, A4, S3, deg, post_layers=1)
    lay = P.PNAConvSimple(f, 128, A4, S3, deg, post_layers=1)
    lay.load_state_dict(ref.state_dict())
    lay = lay.to(dev())
    assert lay._compact(x.to(dev()))
    wout = torch.randn(n, 128, generator=torch.Generator().manual_seed(7))
    xg = x.to(dev()).requires_grad_(True)
    (lay(xg, ei.to(dev())) * wout.to(dev())).sum().backward()
    xr = x.clone().requires_grad_(True)
    (ref(xr, ei) * wout).sum().backward()
    torch.testing.assert_close(xg.grad.cpu(), xr.grad, rtol=1e-3, atol=5e-4)
    for (k, p), (_, p2) in zip(sorted(lay.named_parameters()), sorted(ref.named_parameters())):
        err = float((p.grad.cpu() - p2.grad).norm() / p2.grad.norm().clamp(min=1e-6))
        assert err < 2e-3, f"{k}: relative Frobenius error {err:.2e}"
    # the first post linear's weight gradient (its inputs are the aggregate and the upstream gradient), tighter
    gw, gw2 = lay.post_nn[0].weight.grad.cpu(), ref.post_nn[0].weight.grad
    assert float((gw - gw2).norm() / gw2.norm()) < 1e-4


def _twice(run):
    a, b = run(), run()
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    return a


def test_pnaconvsimple_training_steps_repeat_bit_for_bit(deterministic):
    import pna_b200 as P
    n, f = 4000, 64
    ei = _graph(n, 30000, 8).to(dev())
    x = torch.randn(n, f, generator=torch.Generator().manual_seed(9)).to(dev())
    deg = torch.bincount(torch.bincount(ei[1].cpu(), minlength=n))
    torch.manual_seed(1)
    lay = P.PNAConvSimple(f, 128, A4, S3, deg, post_layers=2).to(dev())
    state = {k: v.clone() for k, v in lay.state_dict().items()}

    def run():
        lay.load_state_dict(state)
        opt = torch.optim.SGD(lay.parameters(), lr=0.1)
        xg = x.clone().requires_grad_(True)
        for _ in range(2):                                          # two training steps
            opt.zero_grad()
            xg.grad = None
            lay(xg, ei).square().mean().backward()
            opt.step()
        return [xg.grad.clone()] + [p.detach().clone() for _, p in sorted(lay.named_parameters())]
    _twice(run)


def test_pnasimplelayer_gradients(deterministic, monkeypatch):
    """DGL-signature simple layer: gradients through the compact path against the library path over the full
    [N, S*A*F] tensor, and bit for bit repeatable."""
    import pna_b200 as P
    from oracle import pna_oracle as O
    n, f = 3000, 64
    ei = _graph(n, 24000, 10)
    avg = O.avg_deg_from_histogram(torch.bincount(torch.bincount(ei[1], minlength=n)))
    avg_d = {k: torch.tensor(v) for k, v in avg.items()}
    torch.manual_seed(2)
    lay = P.PNASimpleLayer(f, 64, "mean max min std", "identity amplification attenuation", avg_d, dropout=0.0,
                           batch_norm=False, residual=True).to(dev())
    gr = P.Graph(ei[0], ei[1], n).to(dev())
    x = torch.randn(n, f, generator=torch.Generator().manual_seed(11)).to(dev())
    wout = torch.randn(n, 64, generator=torch.Generator().manual_seed(12)).to(dev())

    def run():
        lay.zero_grad()
        h = x.clone().requires_grad_(True)
        (lay(gr, h) * wout).sum().backward()
        return [h.grad.clone()] + [p.grad.clone() for _, p in sorted(lay.named_parameters()) if p.grad is not None]
    got = _twice(run)
    monkeypatch.setenv("PNA_B200_TENSOR_LINEAR", "0")              # library GEMMs, scaled copies materialised
    want = run()
    torch.testing.assert_close(got[0], want[0], rtol=1e-4, atol=1e-5)
    for a, b in zip(got[1:], want[1:]):
        assert float((a - b).norm() / b.norm().clamp(min=1e-6)) < 1e-5
