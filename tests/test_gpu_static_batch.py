"""Shuffled mini-batches through a StaticBatch on the H100: the padded CSR build against build_csr, the aggregation
through a padded CSR against the unpadded one and the C oracle, captured training steps replayed over new batches
against eager steps through the same StaticBatch (bit for bit under torch.use_deterministic_algorithms(True)), and eager
static steps against the existing unpadded path."""
import contextlib
import copy
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")     # deterministic cuBLAS under use_deterministic_algorithms

import pna_b200
from pna_b200 import capture, readout, synth
from pna_b200.csr import build_csr

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


# ---- shuffled batches of a pool of graphs ---------------------------------------------------------------------------
class Pool:
    def __init__(self, shape):
        if shape == "zinc":
            self.ei, self.x, self.ng = synth.zinc_like(n_graphs=1500, n_feat=75, seed=7)
        else:
            n_graphs = 400
            self.ei, self.x = synth.superpixel_like(n_graphs=n_graphs, nodes_per_graph=70, k=8, n_feat=75, seed=7)
            self.ng = torch.repeat_interleave(torch.arange(n_graphs), 70)
        G = int(self.ng.max()) + 1
        self.G = G
        gen = torch.Generator().manual_seed(8)
        self.e = torch.randn(self.ei.size(1), 16, generator=gen)
        self.y = torch.randn(G, generator=gen)
        self.snorm = torch.rand(self.x.size(0), 1, generator=gen)
        sizes = torch.bincount(self.ng, minlength=G)
        esizes = torch.bincount(self.ng[self.ei[1]], minlength=G)
        self.caps = (int(sizes.sort(descending=True).values[:128].sum()), int(esizes.sort(descending=True).values[:128].sum()), 128)

    def batches(self, k, seed, lo=80, hi=128):
        gen = torch.Generator().manual_seed(seed)
        for _ in range(k):
            m = int(torch.randint(lo, hi + 1, (1,), generator=gen))
            ids = torch.randperm(self.G, generator=gen)[:m]
            ei, sizes, nid, eid = synth.sub_batch(self.ei, self.ng, ids)
            yield dict(ei=ei, sizes=sizes, x=self.x[nid], e=self.e[eid], snorm=self.snorm[nid], y=self.y[ids])

    def static(self):
        return pna_b200.StaticBatch(*self.caps, device=DEV)


_POOLS = {}


def pool(shape="zinc") -> Pool:
    if shape not in _POOLS:
        _POOLS[shape] = Pool(shape)
    return _POOLS[shape]


def copy_in(sb, b, y_s):
    sb.copy_(src=b["ei"][0].to(DEV), dst=b["ei"][1].to(DEV), batch_num_nodes=b["sizes"],
             ndata={"x": b["x"].to(DEV), "snorm": b["snorm"].to(DEV)}, edata={"e": b["e"].to(DEV)})
    G = b["y"].numel()
    y_s[:G].copy_(b["y"].to(DEV))
    y_s[G:].zero_()


# ---- 1. the build itself -----------------------------------------------------------------------------------------------
def _check_against_unpadded(sb, ei, sizes):
    n, E, G = int(sizes.sum()), ei.size(1), sizes.numel()
    N, Em = sb.max_nodes, sb.max_edges
    ref = build_csr(ei[0].to(DEV), ei[1].to(DEV), n)
    c = sb.csr
    assert torch.equal(c.rowptr[:n + 1], ref.rowptr) and bool((c.rowptr[n:] == E).all())
    assert torch.equal(c.col[:E], ref.col) and torch.equal(c.perm[:E], ref.perm)
    assert bool((c.col[E:] == 0).all())
    assert torch.equal(c.perm[E:].long(), torch.arange(E, Em, device=DEV))
    assert torch.equal(c.in_degree[:n], ref.in_degree) and bool((c.in_degree[n:] == 0).all())
    assert torch.equal(c.dst_of_slot[:E], ref.dst_of_slot) and bool((c.dst_of_slot[E:] == 0).all())
    if ref.n_hubs == 0:
        assert torch.equal(c.light_rowptr[:n + 1], ref.light_rowptr[:n + 1]) and torch.equal(c.light_col[:E], ref.light_col[:E])
    st = sb.check()
    assert st == {"edges": E, "max_degree": ref.max_degree}
    t, rt = c.slot_transposed(N), ref.slot_transposed(n)
    assert torch.equal(t.rowptr[:n + 1], rt.rowptr) and bool((t.rowptr[n:] == E).all())
    assert torch.equal(t.col[:E], rt.col) and torch.equal(t.perm[:E], rt.perm)
    batch = torch.repeat_interleave(torch.arange(G), sizes).to(DEV)
    rr = readout.batch_csr(batch, G)
    assert torch.equal(sb.readout_csr.rowptr[:G + 1], rr.rowptr) and bool((sb.readout_csr.rowptr[G:] == n).all())
    assert torch.equal(sb.readout_csr.col[:n], rr.col)


@pytest.mark.parametrize("shape", ["zinc", "superpixel"])
def test_padded_build_equals_build_csr(shape):
    P = pool(shape)
    sb = P.static()
    for b in P.batches(3, seed=1):
        sb.copy_(src=b["ei"][0].to(DEV), dst=b["ei"][1].to(DEV), batch_num_nodes=b["sizes"])
        sb.build()
        _check_against_unpadded(sb, b["ei"], b["sizes"])


def test_stray_endpoint_sets_the_error_bit():
    P = pool()
    sb = P.static()
    b = next(P.batches(1, seed=2))
    for bad in (sb.max_nodes + 3, -5):
        ei = b["ei"].clone()
        ei[1, 4] = bad
        sb.copy_(src=ei[0].to(DEV), dst=ei[1].to(DEV), batch_num_nodes=b["sizes"]).build()
        with pytest.raises(pna_b200.PnaError, match="outside its range"):
            sb.check()
    ei = b["ei"].clone()
    ei[0, 2] = sb.max_nodes
    sb.copy_(src=ei[0].to(DEV), dst=ei[1].to(DEV), batch_num_nodes=b["sizes"]).build()
    with pytest.raises(pna_b200.PnaError):
        sb.check()
    sb.copy_(src=b["ei"][0].to(DEV), dst=b["ei"][1].to(DEV), batch_num_nodes=b["sizes"]).build()
    sb.check()


def test_padded_build_captures_and_replays_on_new_batches():
    P = pool()
    sb = P.static()
    bs = list(P.batches(4, seed=3))
    sb.copy_(src=bs[0]["ei"][0].to(DEV), dst=bs[0]["ei"][1].to(DEV), batch_num_nodes=bs[0]["sizes"]).build()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with capture.pinned() as keep, torch.cuda.graph(graph):
        sb.build()
    assert sb in keep.objects
    for b in bs[1:]:
        sb.copy_(src=b["ei"][0].to(DEV), dst=b["ei"][1].to(DEV), batch_num_nodes=b["sizes"])
        graph.replay()
        _check_against_unpadded(sb, b["ei"], b["sizes"])


# ---- 2. the aggregation contract ---------------------------------------------------------------------------------------
def test_aggregation_through_the_padded_csr_equals_the_unpadded_csr():
    P = pool()
    sb = P.static()
    avg = {"log": 1.2, "lin": 2.2}
    with _mode(True):
        for b in P.batches(2, seed=4):
            sb.copy_(src=b["ei"][0].to(DEV), dst=b["ei"][1].to(DEV), batch_num_nodes=b["sizes"]).build()
            n, E = int(b["sizes"].sum()), b["ei"].size(1)
            ref = build_csr(b["ei"][0].to(DEV), b["ei"][1].to(DEV), n)
            assert ref.n_hubs == 0
            gen = torch.Generator(device=DEV).manual_seed(5)
            for in_order, rows in ((False, (n, sb.max_nodes)), (True, (E, sb.max_edges))):
                x = torch.randn(rows[0], 64, device=DEV, generator=gen)
                xp = torch.zeros(rows[1], 64, device=DEV)
                xp[:rows[0]] = x
                x.requires_grad_(True)
                xp.requires_grad_(True)
                kw = dict(zero_isolated=True, relu_var=True, messages_in_csr_order=in_order)
                want = pna_b200.pna_aggregate(x, ref, A4, S3, avg, **kw)
                got = pna_b200.pna_aggregate(xp, sb.csr, A4, S3, avg, **kw)
                assert torch.equal(got[:n], want)
                go = torch.randn(want.shape, device=DEV, generator=gen)
                gop = torch.zeros(got.shape, device=DEV)
                gop[:n] = go
                gw, = torch.autograd.grad(want, x, go)
                gg, = torch.autograd.grad(got, xp, gop)
                assert torch.equal(gg[:rows[0]], gw)
                assert bool((gg[rows[0]:] == 0).all())


def test_a_high_degree_row_is_a_light_row_equal_to_the_oracle():
    from oracle import c_oracle
    n, gen = 400, torch.Generator().manual_seed(6)
    src = torch.cat([torch.arange(1, 301), torch.randint(0, n, (900,), generator=gen)])
    dst = torch.cat([torch.zeros(300, dtype=torch.long), torch.randint(1, n, (900,), generator=gen)])
    ei = torch.stack([src, dst])
    split = build_csr(src.to(DEV), dst.to(DEV), n)
    assert split.n_hubs >= 1            # a split row under build_csr
    sb = pna_b200.StaticBatch(n + 50, ei.size(1) + 100, 4, device=DEV)
    sb.copy_(src=src.to(DEV), dst=dst.to(DEV), batch_num_nodes=[n]).build()
    assert sb.check()["max_degree"] == 300
    x = torch.randn(n, 32, generator=gen)
    xp = torch.zeros(sb.max_nodes, 32)
    xp[:n] = x
    avg = {"log": 1.5, "lin": 3.0}
    got = pna_b200.pna_aggregate(xp.to(DEV), sb.csr, A4, ["identity"], avg).cpu()
    want = c_oracle.aggregate(x, ei, A4, ["identity"], avg)
    assert torch.equal(got[:n], want)


# ---- the nets --------------------------------------------------------------------------------------------------------
def _avg(P):
    indeg = torch.bincount(P.ei[1], minlength=P.x.size(0)).float()
    return {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}


class DGLNet(nn.Module):
    def __init__(self, P, edge_features=False, pretrans_layers=1, simple=False, layers=2):
        super().__init__()
        avg = _avg(P)
        if simple:
            self.layers = nn.ModuleList([pna_b200.PNASimpleLayer(75, 75, A4, S3, avg, 0.0, True, True) for _ in range(layers)])
        else:
            self.layers = nn.ModuleList([
                pna_b200.PNALayer(75, 75, A4, S3, avg, 0.0, True, True, towers=5, divide_input=True, residual=True,
                                  pretrans_layers=pretrans_layers, edge_features=edge_features, edge_dim=16)
                for _ in range(layers)])
        self.simple = simple
        self.mlp = nn.Sequential(nn.Linear(75, 32), nn.ReLU(), nn.Linear(32, 1))

    def forward(self, g, x, e, snorm):
        h = x
        for lay in self.layers:
            h = lay(g, h) if self.simple else lay(g, h, e, snorm)
        g.ndata["h"] = h
        return self.mlp(readout.mean_nodes(g, "h")).squeeze(-1)


class PygNet(nn.Module):
    def __init__(self, P, simple=False):
        super().__init__()
        deg = synth.degree_histogram(P.ei[1], P.x.size(0))
        self.convs = nn.ModuleList([
            pna_b200.PNAConvSimple(75, 75, A4, S3, deg, post_layers=1) if simple else
            pna_b200.PNAConv(75, 75, A4, S3, deg, edge_dim=16, towers=5, pre_layers=1, post_layers=1, divide_input=True)
            for _ in range(2)])
        self.bns = nn.ModuleList([nn.BatchNorm1d(75) for _ in range(2)])
        self.lin = nn.Linear(75, 1)

    def forward(self, x, edge_index, e, batch, n_graphs, csr=None, sb=None):
        h = x
        for conv, bn in zip(self.convs, self.bns):
            h = conv(h, edge_index, e, csr=csr)
            h = F.relu(sb.batch_norm(bn, h) if sb is not None else bn(h))
        return self.lin(readout.global_mean_pool(h, batch, n_graphs)).squeeze(-1)


class ReadoutNet(nn.Module):
    def __init__(self, P):
        super().__init__()
        self.lin = nn.Linear(75, 32)
        self.out = nn.Linear(5 * 32, 1)

    def forward(self, g, x, batch, n_graphs):
        h = self.lin(x)
        g.ndata["h"] = h
        r = torch.cat([readout.sum_nodes(g, "h"), readout.max_nodes(g, "h"), readout.global_add_pool(h, batch, n_graphs),
                       readout.global_mean_pool(h, batch, n_graphs), readout.global_max_pool(h, batch, n_graphs)], 1)
        return self.out(r).squeeze(-1)


def _case(name):
    P = pool()
    torch.manual_seed(0)
    if name.startswith("dgl"):
        m = DGLNet(P, edge_features="edge" in name, pretrans_layers=2 if "pre2" in name else 1, simple="simple" in name)
        static = lambda m, sb: m(sb, sb.ndata["x"], sb.edata["e"], sb.ndata["snorm"])

        def plain(m, b):
            g = pna_b200.Graph(b["ei"][0], b["ei"][1], int(b["sizes"].sum()), batch_num_nodes=b["sizes"].tolist()).to(DEV)
            return m(g, b["x"].to(DEV), b["e"].to(DEV), b["snorm"].to(DEV))
    elif name.startswith("pyg"):
        m = PygNet(P, simple="simple" in name)
        static = lambda m, sb: m(sb.ndata["x"], sb.edge_index, None if m.convs[0].__class__.__name__ == "PNAConvSimple"
                                 else sb.edata["e"], sb.batch, sb.max_graphs, csr=sb.csr, sb=sb)

        def plain(m, b):
            G = b["sizes"].numel()
            batch = torch.repeat_interleave(torch.arange(G), b["sizes"]).to(DEV)
            e = None if "simple" in name else b["e"].to(DEV)
            return m(b["x"].to(DEV), b["ei"].to(DEV), e, batch, G)
    else:
        m = ReadoutNet(P)
        static = lambda m, sb: m(sb, sb.ndata["x"], sb.batch, sb.max_graphs)

        def plain(m, b):
            G = b["sizes"].numel()
            g = pna_b200.Graph(b["ei"][0], b["ei"][1], int(b["sizes"].sum()), batch_num_nodes=b["sizes"].tolist()).to(DEV)
            return m(g, b["x"].to(DEV), torch.repeat_interleave(torch.arange(G), b["sizes"]).to(DEV), G)
    return P, m.to(DEV).train(), static, plain


CASES = ["dgl", "dgl_edge", "dgl_edge_pre2", "dgl_simple", "pyg_edge", "pyg_simple", "readouts"]


def _masked_loss(out, sb, y_s):
    return (((out - y_s) ** 2) * sb.graph_mask).sum() / sb.counts[2].float()


def _same(got, want, exact, what, rel=1e-4):
    if exact:
        assert torch.equal(got, want), f"{what}: differs by {(got - want).abs().max().item():.3e}"
    else:
        bar = rel * want.abs().max().item() + 1e-6
        err = (got - want).abs().max().item()
        assert err <= bar, f"{what}: differs by {err:.3e} (bar {bar:.3e})"


def _replay_vs_eager(name, exact, amp=None, n_batches=5):
    P, m, static, _ = _case(name)
    sb = P.static()
    y_s = torch.zeros(sb.max_graphs, device=DEV)
    params = list(m.parameters())

    def step():
        sb.build()
        ctx = torch.autocast("cuda", dtype=amp, cache_enabled=False) if amp is not None else contextlib.nullcontext()
        with ctx:
            out = static(m, sb).float()
        loss = _masked_loss(out, sb, y_s)
        return (out.detach(), loss.detach()) + tuple(torch.autograd.grad(loss, params))

    bs = list(P.batches(n_batches + 1, seed=9, lo=60))
    copy_in(sb, bs[0], y_s)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with capture.pinned() as keep, torch.cuda.graph(graph):
        s_res = step()
    bufs = list(m.buffers())
    for k, b in enumerate(bs[1:]):
        copy_in(sb, b, y_s)
        before = [t.clone() for t in bufs]
        graph.replay()
        got = [t.clone() for t in s_res]
        got_bufs = [t.clone() for t in bufs]
        for t, s in zip(bufs, before):
            t.copy_(s)
        want = step()
        G = b["y"].numel()
        _same(got[0][:G], want[0][:G], exact, f"batch {k} output")
        for i, (a, w) in enumerate(zip(got[1:], want[1:])):
            _same(a, w, exact, f"batch {k} loss / gradient {i}")
        for i, (a, w) in enumerate(zip(got_bufs, bufs)):
            _same(a.float(), w.float(), exact, f"batch {k} buffer {i}")
    assert sb in keep.objects


# ---- 3. replay equals eager static -------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_replay_equals_eager_static_step_bit_for_bit(name):
    with _mode(True):
        _replay_vs_eager(name, exact=True)


@pytest.mark.parametrize("name", ["dgl_edge_pre2", "pyg_edge"])
def test_replay_equals_eager_static_step_in_atomic_mode(name):
    _replay_vs_eager(name, exact=False)


def test_bf16_autocast_replay_equals_eager_static_step():
    with _mode(True):
        _replay_vs_eager("dgl", exact=True, amp=torch.bfloat16, n_batches=3)


# ---- 4. static equals unpadded -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", CASES)
def test_eager_static_step_equals_the_unpadded_step(name):
    P, m, static, plain = _case(name)
    twin = copy.deepcopy(m)
    sb = P.static()
    y_s = torch.zeros(sb.max_graphs, device=DEV)
    for k, b in enumerate(P.batches(2, seed=10)):
        copy_in(sb, b, y_s)
        sb.build()
        out = static(m, sb)
        loss = _masked_loss(out, sb, y_s)
        grads = torch.autograd.grad(loss, list(m.parameters()))
        out_r = plain(twin, b)
        loss_r = ((out_r - b["y"].to(DEV)) ** 2).mean()
        grads_r = torch.autograd.grad(loss_r, list(twin.parameters()))
        G = b["y"].numel()
        _same(out[:G].detach(), out_r.detach(), False, f"batch {k} output")
        _same(loss.detach(), loss_r.detach(), False, f"batch {k} loss")
        # a weight gradient sums over every node row, and two batch norm backwards (cuDNN's against autograd of the masked
        # statistics) reorder what reaches it: PNAConvSimple's first post Linear measured 3.4e-4 of its largest entry
        for (pn, _), a, w in zip(m.named_parameters(), grads, grads_r):
            _same(a, w, False, f"batch {k} gradient of {pn}", rel=1e-3)
        for (bn_, a), w in zip(m.named_buffers(), twin.buffers()):
            _same(a.float(), w.float(), False, f"batch {k} buffer {bn_}")


# ---- 5. training loops -------------------------------------------------------------------------------------------------
def _captured_loop(P, m, static, opt, bs):
    sb = P.static()
    y_s = torch.zeros(sb.max_graphs, device=DEV)

    def train_step():
        opt.zero_grad(set_to_none=True)
        sb.build()
        _masked_loss(static(m, sb).float(), sb, y_s).backward()
        opt.step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for b in bs[:2]:
            copy_in(sb, b, y_s)
            train_step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    opt.zero_grad(set_to_none=True)
    with capture.pinned() as keep, torch.cuda.graph(graph):
        sb.build()
        _masked_loss(static(m, sb).float(), sb, y_s).backward()
        opt.step()
    for b in bs[2:]:
        copy_in(sb, b, y_s)
        graph.replay()
    torch.cuda.synchronize()
    return keep


def test_captured_adam_loop_equals_the_eager_static_loop():
    with _mode(True):
        P, m, static, _ = _case("dgl_edge")
        twin = copy.deepcopy(m)
        bs = list(P.batches(20, seed=11, lo=60))
        keep = _captured_loop(P, m, static, torch.optim.Adam(m.parameters(), lr=1e-3, capturable=True), bs)
        opt_t = torch.optim.Adam(twin.parameters(), lr=1e-3, capturable=True)
        sb = P.static()
        y_s = torch.zeros(sb.max_graphs, device=DEV)
        for b in bs:
            copy_in(sb, b, y_s)
            opt_t.zero_grad(set_to_none=True)
            sb.build()
            _masked_loss(static(twin, sb).float(), sb, y_s).backward()
            opt_t.step()
        for (name, p), q in zip(m.named_parameters(), twin.parameters()):
            assert torch.equal(p, q), f"{name}: captured loop differs by {(p - q).abs().max().item():.3e}"
        for (name, a), w in zip(m.named_buffers(), twin.buffers()):
            assert torch.equal(a, w), name
        assert keep.objects


def test_captured_sgd_loop_ends_near_the_eager_unpadded_loop():
    P, m, static, plain = _case("dgl_edge")
    twin = copy.deepcopy(m)
    bs = list(P.batches(20, seed=12, lo=60))
    _captured_loop(P, m, static, torch.optim.SGD(m.parameters(), lr=1e-3), bs)
    opt_t = torch.optim.SGD(twin.parameters(), lr=1e-3)
    for b in bs:
        opt_t.zero_grad(set_to_none=True)
        ((plain(twin, b) - b["y"].to(DEV)) ** 2).mean().backward()
        opt_t.step()
    for (name, p), q in zip(m.named_parameters(), twin.parameters()):
        _same(p.detach(), q.detach(), False, name)
