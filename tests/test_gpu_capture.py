"""CUDA-graph capture of the layers on the H100: every layer family is warmed up eagerly, its forward (and backward) is
captured with torch.cuda.graph inside pna_b200.capture.pinned(), replayed with new feature values copied into the static
inputs and new parameter values, and compared with an eager step on the same values.  Under
torch.use_deterministic_algorithms(True) every kernel path is atomics-free and the comparison is bit for bit; in the default
(atomic) backward mode it is held to a bar relative to the largest entry."""
import contextlib
import copy
import os

import pytest
import torch

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")     # deterministic cuBLAS under use_deterministic_algorithms

import pna_b200
from pna_b200 import _lib, capture, dense, edge_mlp, linear, readout, synth

DEV = torch.device("cuda:0")
A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]
pytestmark = pytest.mark.gpu


@contextlib.contextmanager
def _mode(deterministic):
    torch.use_deterministic_algorithms(deterministic)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(False)


# ---- the layer families -------------------------------------------------------------------------------------------
def _pyg_simple():
    ei, x = synth.arxiv_like(n_nodes=3000, n_edges=30000, n_feat=64, seed=1)
    torch.manual_seed(0)
    m = pna_b200.PNAConvSimple(64, 64, A4, S3, synth.degree_histogram(ei[1], 3000), post_layers=2).to(DEV)
    eid = ei.to(DEV)
    return m, {"x": x.to(DEV)}, lambda m, i: m(i["x"], eid)


def _pyg(edge_dim=None, pre_layers=1, post_layers=2):
    ei, x = synth.arxiv_like(n_nodes=3000, n_edges=30000, n_feat=60, seed=2)
    torch.manual_seed(0)
    m = pna_b200.PNAConv(60, 60, A4, S3, synth.degree_histogram(ei[1], 3000), edge_dim=edge_dim, towers=4,
                         pre_layers=pre_layers, post_layers=post_layers, divide_input=True).to(DEV)
    eid = ei.to(DEV)
    inputs = {"x": x.to(DEV)}
    if edge_dim:
        inputs["e"] = torch.randn(ei.size(1), edge_dim, device=DEV)
    return m, inputs, lambda m, i: m(i["x"], eid, i.get("e"))


def _zinc_batch():
    ei, x, _ = synth.zinc_like(n_graphs=128, n_feat=75)
    n = x.size(0)
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    return ei, x, n, avg


def _dgl(edge_features=False, pretrans_layers=1):
    ei, x, n, avg = _zinc_batch()
    torch.manual_seed(0)
    m = pna_b200.PNALayer(75, 75, A4, S3, avg, 0.0, True, True, towers=5, divide_input=True, residual=True,
                          pretrans_layers=pretrans_layers, edge_features=edge_features, edge_dim=16).to(DEV)
    g = pna_b200.Graph(ei[0], ei[1], n).to(DEV)
    inputs = {"x": x.to(DEV), "snorm": torch.rand(n, 1, device=DEV)}
    if edge_features:
        inputs["e"] = torch.randn(ei.size(1), 16, device=DEV)
    return m, inputs, lambda m, i: m(g, i["x"], i.get("e"), i["snorm"])


def _dgl_simple():
    ei, x, n, avg = _zinc_batch()
    torch.manual_seed(0)
    m = pna_b200.PNASimpleLayer(75, 75, A4, S3, avg, 0.0, True, True).to(DEV)
    g = pna_b200.Graph(ei[0], ei[1], n).to(DEV)
    return m, {"x": x.to(DEV)}, lambda m, i: m(g, i["x"])


def _dense(aggregators, pretrans_layers=1, self_loop=False):
    B, N, F = 128, 32, 16                                   # the multitask benchmark's batch shape
    gen = torch.Generator().manual_seed(3)
    adj = (torch.rand(B, N, N, generator=gen) < 0.15).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float().to(DEV)
    torch.manual_seed(0)
    m = dense.PNALayer(F, F, aggregators, ["identity", "amplification", "attenuation"], {"log": 1.6, "lin": 4.8}, towers=2,
                       pretrans_layers=pretrans_layers, self_loop=self_loop, divide_input=True).to(DEV)
    return m, {"x": torch.randn(B, N, F, generator=gen).to(DEV)}, lambda m, i: m(i["x"], adj)


class _Readouts(torch.nn.Module):
    def __init__(self, n_graphs):
        super().__init__()
        self.lin = torch.nn.Linear(75, 32)
        self.n_graphs = n_graphs

    def forward(self, g, x, batch):
        h = self.lin(x)
        g.ndata["h"] = h
        return torch.cat([readout.global_add_pool(h, batch, self.n_graphs), readout.global_mean_pool(h, batch, self.n_graphs),
                          readout.global_max_pool(h, batch, self.n_graphs), readout.sum_nodes(g, "h"),
                          readout.max_nodes(g, "h")], 1)


def _readouts():
    ei, x, n, _ = _zinc_batch()
    per = n // 128
    sizes = [per] * 127 + [n - 127 * per]
    g = pna_b200.Graph(ei[0], ei[1], n, batch_num_nodes=sizes).to(DEV)
    batch = torch.repeat_interleave(torch.arange(128), torch.tensor(sizes)).to(DEV)
    torch.manual_seed(0)
    m = _Readouts(128).to(DEV)
    return m, {"x": x.to(DEV)}, lambda m, i: m(g, i["x"], batch)


CASES = {
    "pyg_simple": _pyg_simple,
    "pyg_towers": lambda: _pyg(post_layers=1),          # without autograd: every GEMM on the tensor cores
    "pyg_edge_pre1": lambda: _pyg(edge_dim=8, pre_layers=1),
    "pyg_edge_pre2": lambda: _pyg(edge_dim=8, pre_layers=2),
    "dgl": lambda: _dgl(),
    "dgl_edge_pre2": lambda: _dgl(edge_features=True, pretrans_layers=2),
    "dgl_simple": _dgl_simple,
    # the dense registry's kernel paths across the three (at most PNA_MAX_AGGR = 6 names per layer)
    "dense_all": lambda: _dense(["mean", "max", "std", "var", "moment3", "softmax"]),
    "dense_pre2": lambda: _dense(["mean", "max", "min", "std", "identity"], pretrans_layers=2),
    "dense_self_loop": lambda: _dense(["sum", "min", "softmin", "normalised_mean", "identity"], self_loop=True),
    "readouts": _readouts,
}


# ---- capture, replay, compare -------------------------------------------------------------------------------------
def _same(got, want, exact, what):
    if exact:
        assert torch.equal(got, want), f"{what}: replay differs from eager by {(got - want).abs().max().item():.3e}"
    else:
        bar = 1e-4 * want.abs().max().item() + 1e-6
        err = (got - want).abs().max().item()
        assert err <= bar, f"{what}: replay differs from eager by {err:.3e} (bar {bar:.3e})"


def _replay_matches_eager(model, inputs, run, train, exact, amp=None, rounds=3):
    """Warm up on a side stream, capture one step (forward, and backward when ``train``), then per round: new feature
    values and new parameter values in place, replay, and the same step eagerly.  Returns the pinned handle."""
    model.train(train)
    params = [p for p in model.parameters()]
    feats = [k for k, v in inputs.items() if v.is_floating_point() and k != "snorm"]
    if train:
        inputs["x"].requires_grad_(True)
    leaves = params + [inputs["x"]] if train else []

    def step():
        ctx = torch.autocast("cuda", dtype=amp, cache_enabled=False) if amp is not None else contextlib.nullcontext()
        with ctx, torch.set_grad_enabled(train):
            out = run(model, inputs).float()
        proj = torch.linspace(-1.0, 1.0, out.numel(), device=DEV).view(out.shape)
        grads = torch.autograd.grad((out * proj).sum(), leaves, allow_unused=True) if train else ()
        return out.detach(), grads

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with capture.pinned() as keep:
        with torch.cuda.graph(graph):
            s_out, s_grads = step()
    gen = torch.Generator(device=DEV).manual_seed(11)
    for r in range(rounds):
        with torch.no_grad():
            for k in feats:
                inputs[k].copy_(torch.randn(inputs[k].shape, device=DEV, generator=gen))
            for p in params:                                # weights change between replays: the packs must follow
                p.add_(torch.randn(p.shape, device=DEV, generator=gen), alpha=1e-2)
        graph.replay()
        got = (s_out.clone(), [None if t is None else t.clone() for t in s_grads])
        want = step()
        _same(got[0], want[0], exact, f"round {r} output")
        for i, (a, b) in enumerate(zip(got[1], want[1])):
            assert (a is None) == (b is None)
            if a is not None:
                _same(a, b, exact, f"round {r} gradient {i}")
    return keep


@pytest.fixture
def fused_everywhere(monkeypatch):
    """The fused edge-message kernels in training steps at these small shapes too (that gate is set by speed, not by
    what is capturable)."""
    monkeypatch.setattr(edge_mlp, "FUSED_TRAINING_MIN_EDGES", 0)


@pytest.mark.parametrize("train", [False, True], ids=["forward", "train"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_replay_is_bit_identical_in_deterministic_mode(case, train, fused_everywhere):
    with _mode(True):
        model, inputs, run = CASES[case]()
        keep = _replay_matches_eager(model, inputs, run, train, exact=True)
    assert keep.objects                        # the per-graph state the capture touched was recorded


@pytest.mark.parametrize("case", ["pyg_towers", "pyg_edge_pre2", "dgl", "dense_all"])
def test_replay_matches_eager_in_atomic_mode(case, fused_everywhere):
    model, inputs, run = CASES[case]()
    _replay_matches_eager(model, inputs, run, True, exact=False)


@pytest.mark.parametrize("case", ["pyg_towers", "dgl"])
def test_compact_tower_path_replays(case, fused_everywhere, monkeypatch):
    monkeypatch.setattr(linear, "TOWERS_COMPACT_MIN_ROWS", 0)
    with _mode(True):
        model, inputs, run = CASES[case]()
        _replay_matches_eager(model, inputs, run, True, exact=True)


@pytest.mark.parametrize("train", [False, True], ids=["forward", "train"])
@pytest.mark.parametrize("case", ["pyg_towers", "pyg_edge_pre2", "dgl_edge_pre2", "dense_pre2", "readouts"])
def test_replay_under_bf16_autocast(case, train, fused_everywhere):
    with _mode(True):
        model, inputs, run = CASES[case]()
        _replay_matches_eager(model, inputs, run, train, exact=True, amp=torch.bfloat16)


# ---- whole training steps -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["pyg_edge_pre2", "dgl", "dense_all"])
def test_captured_training_loop_matches_eager_loop(case, fused_everywhere):
    """forward, backward and a capturable Adam step in one graph: after several replays the parameters equal those of the
    same loop run eagerly, bit for bit (stale weight packs would show here)."""
    with _mode(True):
        model, inputs, run = CASES[case]()
        model.train()
        twin = copy.deepcopy(model)
        opt = torch.optim.Adam(model.parameters(), lr=1e-2, capturable=True)
        opt_t = torch.optim.Adam(twin.parameters(), lr=1e-2, capturable=True)
        gen = torch.Generator(device=DEV).manual_seed(5)
        batches = [{k: (torch.randn(v.shape, device=DEV, generator=gen) if v.is_floating_point() and k != "snorm" else v)
                    for k, v in inputs.items()} for _ in range(6)]

        def loss_of(m, i):
            out = run(m, i).float()
            return (out * torch.linspace(-1.0, 1.0, out.numel(), device=DEV).view(out.shape)).sum()

        def train_step(m, o, i):
            o.zero_grad(set_to_none=True)
            loss_of(m, i).backward()
            o.step()

        static = {k: v.clone() for k, v in inputs.items()}
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for b in batches[:2]:
                for k in static:
                    static[k].copy_(b[k])
                train_step(model, opt, static)
        torch.cuda.current_stream().wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        opt.zero_grad(set_to_none=True)
        with capture.pinned() as keep:
            with torch.cuda.graph(graph):
                loss_of(model, static).backward()
                opt.step()
        for b in batches[2:]:
            for k in static:
                static[k].copy_(b[k])
            graph.replay()
        for b in batches:
            train_step(twin, opt_t, b)
        torch.cuda.synchronize()
        for (name, p), q in zip(model.named_parameters(), twin.parameters()):
            assert torch.equal(p, q), f"{name}: captured loop differs from eager loop by {(p - q).abs().max().item():.3e}"
        assert keep.objects


# ---- pinning --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["pyg_simple", "dense_all", "readouts"])
def test_replay_survives_cache_eviction(case, fused_everywhere):
    """After more graphs than any cache holds have passed through the layers (and their memory has been reused), the
    captured graph still reads its own CSRs: replay equals eager."""
    with _mode(True):
        model, inputs, run = CASES[case]()
        model.eval()
        with torch.no_grad():
            run(model, inputs)
            graph = torch.cuda.CUDAGraph()
            with capture.pinned() as keep:
                with torch.cuda.graph(graph):
                    s_out = run(model, inputs)
        if case == "pyg_simple":
            for k in range(20):
                ei, x = synth.arxiv_like(n_nodes=3000, n_edges=30000, n_feat=64, seed=100 + k)
                with torch.no_grad():
                    model(x.to(DEV), ei.to(DEV))
        elif case == "dense_all":
            for k in range(20):
                adj = (torch.rand(128, 32, 32, device=DEV) < 0.3).float()
                with torch.no_grad():
                    model(inputs["x"], adj)
        else:
            for k in range(20):
                b = torch.randint(0, 128, (inputs["x"].size(0),), device=DEV).sort().values
                with torch.no_grad():
                    readout.global_add_pool(inputs["x"][:, :32].contiguous(), b, 128)
        assert len(pna_b200.csr._CACHE) <= pna_b200.csr._CACHE_SIZE and len(dense._CACHE) <= 9 and len(readout._CACHE) <= 8
        junk = [torch.full((1 << 20,), 7.0, device=DEV) for _ in range(64)]       # reuse whatever was freed
        with torch.no_grad():
            inputs["x"].copy_(torch.randn_like(inputs["x"]))
            graph.replay()
            want = run(model, inputs)
        assert torch.equal(s_out, want)
        del junk, keep


# ---- refusals -------------------------------------------------------------------------------------------------------
def test_capture_error_for_an_unseen_graph_then_capture_works():
    model, inputs, run = CASES["pyg_simple"]()
    model.eval()
    ei, _ = synth.arxiv_like(n_nodes=3000, n_edges=30000, n_feat=64, seed=77)
    unseen = ei.to(DEV)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad():
        with pytest.raises(pna_b200.CaptureError, match="run one eager step on this graph first"):
            with torch.cuda.graph(graph):
                model(inputs["x"], unseen)
        assert not torch.cuda.is_current_stream_capturing()
        run(model, inputs)                                   # eager, then a normal capture
        g2 = torch.cuda.CUDAGraph()
        with capture.pinned() as keep:
            with torch.cuda.graph(g2):
                s_out = run(model, inputs)
        g2.replay()
        assert torch.equal(s_out, run(model, inputs))
    del keep


def test_pna_csr_build_returns_capturing_status(monkeypatch):
    src = torch.randint(0, 100, (500,), device=DEV)
    dst = torch.randint(0, 100, (500,), device=DEV)
    pna_b200.build_csr(src, dst, 100)                        # loads the library, warms the allocator
    monkeypatch.setattr(capture, "guard", lambda *a, **k: None)   # let the call reach the C library inside the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        with pytest.raises(pna_b200.PnaError) as err:
            pna_b200.build_csr(src, dst, 100)
    assert err.value.status == _lib.PNA_ERR_CAPTURING
    assert not torch.cuda.is_current_stream_capturing()
    assert pna_b200.build_csr(src, dst, 100).n_edges == 500
