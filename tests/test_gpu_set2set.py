"""Set2Set / S2SReadout on the GPU (pna_set2set_fwd / _bwd and the weight-gradient GEMMs).

Accuracy bar, per output and gradient tensor: max|kernel - f64| <= 4 max|torch_fp32 - f64| + 64 * 2^-24 max|f64|, where f64
is the float64 restatement (tests/set2set_ref.py) and torch_fp32 the reference's loop in torch ops in fp32 on the CPU (so no
TF32 loosens the bar).  Also: the reference's golden outputs and gradients, large logits, bit-identical repeats, a captured
training step against an eager one, bf16 autocast and the refusals."""
import os
import sys

import pytest
import torch

import pna_b200

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import set2set_ref as R  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "s2s_readout.pt")


def within_bar(name, kernel, f64, fp32):
    k, w, t = kernel.detach().double().cpu(), f64.detach().double().cpu(), fp32.detach().double().cpu()
    assert torch.isfinite(k).all(), name
    err, ref_err = (k - w).abs().max().item(), (t - w).abs().max().item()
    bar = 4 * ref_err + 64 * 2.0 ** -24 * w.abs().max().item()
    assert err <= bar, f"{name}: max|kernel - f64| = {err:.3e} > bar {bar:.3e} (torch fp32: {ref_err:.3e})"


def kernel_run(mod, x, w):
    xg = x.to(DEV).requires_grad_(True)
    mod.zero_grad(set_to_none=True)
    out = mod(xg)
    (out * w.to(DEV)).sum().backward()
    grads = {"x": xg.grad}
    grads.update({k: p.grad for k, p in mod.named_parameters() if p.grad is not None})
    return out.detach(), grads


def one_case(B, N, D, steps, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    torch.manual_seed(seed)
    lstm = torch.nn.LSTM(2 * D, D, batch_first=True)
    x = torch.randn(B, N, D, generator=g) * scale
    w = torch.randn(B, 2 * D, generator=g)
    # torch fp32 on the CPU: the reference's loop
    xc = x.clone().requires_grad_(True)
    out32 = R.torch_loop(xc, steps, lstm)
    params = [getattr(lstm, p) for p in R.PARAMS]
    g32 = dict(zip(("x",) + R.PARAMS, torch.autograd.grad((out32 * w).sum(), [xc] + params)))
    # float64 restatement
    p64 = [p.detach().double() for p in params]
    out64, recs = R.forward(x.double(), steps, *p64)
    g64 = R.backward(x.double(), p64[0], p64[1], recs, w.double())
    # the kernels
    mod = pna_b200.Set2Set(D, steps=steps).to(DEV)
    mod.load_state_dict({"lstm." + k: v for k, v in lstm.state_dict().items()})
    out, gk = kernel_run(mod, x, w)
    within_bar("out", out, out64, out32)
    within_bar("x", gk["x"], g64["x"], g32["x"])
    for p in R.PARAMS:
        within_bar(p, gk["lstm." + p], g64[p], g32[p])
    return out, gk


SHAPES = [  # (B, N, D, steps): D in {1, 16, 17, 66, 128}, N in {1, 2, 32, 100}, steps in {N, 1, 3, 2N}, B in {1, 128, 300}
    (1, 1, 1, None), (128, 2, 1, 3), (128, 100, 1, 200), (300, 100, 1, None),
    (128, 32, 16, None), (128, 32, 16, 1), (128, 32, 16, 3), (128, 32, 16, 64), (300, 32, 16, None), (128, 100, 16, None),
    (1, 2, 17, 3), (128, 32, 17, None), (300, 1, 17, 2),
    (128, 32, 66, None), (300, 2, 66, 4), (1, 100, 66, 1), (1, 32, 66, 64),
    (128, 100, 128, None), (1, 32, 128, 3), (300, 1, 128, 2),
]


@pytest.mark.parametrize("B,N,D,steps", SHAPES)
def test_kernel_within_the_bar(B, N, D, steps):
    one_case(B, N, D, steps, seed=B + 7 * N + 31 * D + (steps or 0))


@pytest.mark.parametrize("D", [4, 16])
def test_large_logits(D):
    """|x . q| around 10^3: the softmax is only finite because the maximum is subtracted."""
    B, N = 64, 32
    out, _ = one_case(B, N, D, None, seed=5 + D, scale=4000.0 / D ** 0.5)
    assert out.abs().max().item() > 100


@pytest.mark.parametrize("name", sorted(torch.load(GOLDEN)))
def test_golden_readout(name):
    """Reference state_dicts load into the pna_b200 modules and give the reference's outputs and gradients within the bar
    (the reference's own fp32 autograd is the fp32 yardstick)."""
    case = torch.load(GOLDEN)[name]
    mod = (pna_b200.S2SReadout(**case["ctor"]) if case["kind"] == "s2s" else pna_b200.Set2Set(**case["ctor"]))
    mod.load_state_dict(case["state_dict"])
    mod = mod.to(DEV).train(case["train"])
    out, gk = kernel_run(mod, case["x"], case["w"])
    out64, g64 = R.readout(case)
    within_bar("out", out, out64, case["out"])
    for k, want in case["grads"].items():
        within_bar(k, gk[k], g64[k], want)


def _step(mod, x, w):
    out, g = kernel_run(mod, x, w)
    return [out] + [g[k].clone() for k in sorted(g)]


@pytest.mark.parametrize("deterministic", [False, True])
def test_forward_and_backward_repeat_bit_for_bit(deterministic, monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.manual_seed(3)
    mod = pna_b200.S2SReadout(66, 16, 3, final_activation="LeakyReLU").to(DEV)
    x, w = torch.randn(128, 32, 66), torch.randn(128, 3)
    prev = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(deterministic)
    try:
        a, b = _step(mod, x, w), _step(mod, x, w)
    finally:
        torch.use_deterministic_algorithms(prev)
    assert all(torch.equal(u, v) for u, v in zip(a, b))


def test_captured_training_step_replays_like_eager(monkeypatch):
    monkeypatch.setenv("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    torch.manual_seed(4)
    mod = pna_b200.S2SReadout(16, 16, 3, final_activation="LeakyReLU").to(DEV).train()
    params = list(mod.parameters())
    g = torch.Generator().manual_seed(9)
    sx, sw = torch.randn(128, 32, 16, device=DEV), torch.randn(128, 3, device=DEV)

    def body():
        for p in params:
            p.grad = None if p.grad is None else p.grad.zero_()
        out = mod(sx)
        (out * sw).sum().backward()
        return out

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            body()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = body()
    for k in range(3):
        x = torch.randn(128, 32, 16, generator=g)
        weights = [torch.randn(p.shape, generator=g) * 0.3 for p in params]
        with torch.no_grad():
            sx.copy_(x)
            for p, v in zip(params, weights):
                p.copy_(v)
        graph.replay()
        replay = [static_out.clone()] + [p.grad.clone() for p in params]
        eager = [body().detach()] + [p.grad.clone() for p in params]
        assert all(torch.equal(u, v) for u, v in zip(replay, eager)), k


def test_bf16_autocast_upcasts_at_the_boundary():
    torch.manual_seed(6)
    s = pna_b200.Set2Set(16).to(DEV)
    x = torch.randn(32, 20, 16, device=DEV).bfloat16()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = s(x)
    assert out.dtype == torch.float32
    assert torch.equal(out, s(x.float()))
    xg = x.clone().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        s(xg).sum().backward()
    assert xg.grad.dtype == torch.bfloat16 and torch.isfinite(xg.grad.float()).all()


def test_refusals_and_empty_inputs():
    s = pna_b200.Set2Set(128).to(DEV)
    with pytest.raises(NotImplementedError):
        s(torch.randn(2, 129, 128, device=DEV))                    # N * D > 16384
    with pytest.raises(NotImplementedError):
        pna_b200.Set2Set(129).to(DEV)(torch.randn(2, 3, 129, device=DEV))
    with pytest.raises(TypeError):
        s(torch.randn(2, 3, 128, device=DEV).half())               # fp16 outside autocast
    assert torch.equal(s(torch.randn(0, 5, 128, device=DEV)), torch.zeros(0, 256, device=DEV))
    assert torch.equal(s(torch.randn(3, 0, 128, device=DEV)), torch.zeros(3, 256, device=DEV))
    with pytest.raises(NotImplementedError):
        pna_b200.Set2Set(8, steps=2).to(DEV)(torch.randn(3, 0, 8, device=DEV))


def test_inference_saves_nothing_and_matches_training_forward():
    torch.manual_seed(8)
    s = pna_b200.Set2Set(16).to(DEV)
    x = torch.randn(128, 32, 16, device=DEV)
    with torch.no_grad():
        a = s(x)
    b = s(x.requires_grad_(True))
    assert a.grad_fn is None and torch.equal(a, b.detach())
