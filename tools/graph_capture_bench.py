"""Eager steps against CUDA-graph replays of the same steps, alternated in one run.

For each shape, a training step (forward, backward and a capturable Adam step) and an inference forward, each run eagerly
and as a replay of a graph captured with torch.cuda.graph inside pna_b200.capture.pinned(); the features are copied into the
static inputs before every step in both arms.  Median CUDA-event time per step over alternated rounds.  Prints the card
and its power limit, then one JSON line per shape.

    python tools/graph_capture_bench.py [--rounds 5] [--steps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pna_b200  # noqa: E402
from pna_b200 import capture, dense, readout, synth  # noqa: E402

AGGRS = ["mean", "max", "min", "std"]
SCALERS = ["identity", "amplification", "attenuation"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def timed(fn, steps):
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    t.record()
    torch.cuda.synchronize()
    return s.elapsed_time(t) / steps


class DenseStack(torch.nn.Module):
    """Four dense PNALayers at the multitask benchmark's shape (B=128 graphs of N=32 nodes, F=16, towers=2)."""

    def __init__(self, f=16):
        super().__init__()
        self.layers = torch.nn.ModuleList([dense.PNALayer(f, f, AGGRS, SCALERS, {"log": 1.6, "lin": 4.8}, towers=2)
                                           for _ in range(4)])

    def forward(self, x, adj):
        for lay in self.layers:
            x = torch.relu(lay(x, adj))
        return x


def dense_multitask():
    B, N, F = 128, 32, 16
    g = torch.Generator().manual_seed(3)
    adj = (torch.rand(B, N, N, generator=g) < 0.15).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float().cuda()
    torch.manual_seed(0)
    net = DenseStack(F).cuda()
    return net, torch.randn(B, N, F, generator=g).cuda(), lambda x: net(x, adj)


class DglNet(torch.nn.Module):
    """Four DGL PNALayers (75 -> 70, then 70 -> 70; towers=5, batch and graph norm, residual) and a sum readout."""

    def __init__(self, avg):
        super().__init__()
        dims = [75, 70, 70, 70, 70]
        self.layers = torch.nn.ModuleList([
            pna_b200.PNALayer(dims[k], dims[k + 1], AGGRS, SCALERS, avg, 0.0, True, True, towers=5, divide_input=True,
                              residual=True) for k in range(4)])

    def forward(self, g, h, snorm):
        for lay in self.layers:
            h = lay(g, h, None, snorm)
        g.ndata["h"] = h
        return readout.sum_nodes(g, "h")


def dgl_zinc_batch():
    ei, x, _ = synth.zinc_like(n_graphs=128, n_feat=75)
    n = x.size(0)
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    per = n // 128
    g = pna_b200.Graph(ei[0], ei[1], n, batch_num_nodes=[per] * 127 + [n - 127 * per]).to("cuda")
    snorm = torch.ones(n, 1, device="cuda")
    torch.manual_seed(0)
    net = DglNet(avg).cuda()
    return net, x.cuda(), lambda h: net(g, h, snorm)


def pyg_config2():
    ei, x = synth.arxiv_like(n_feat=128, seed=0)
    n = x.size(0)
    torch.manual_seed(0)
    conv = pna_b200.PNAConvSimple(128, 128, AGGRS, SCALERS, synth.degree_histogram(ei[1], n)).cuda()
    eid = ei.cuda()
    return conv, x.cuda(), lambda xx: conv(xx, eid)


def measure(name, make, rounds, steps):
    net, x, call = make()
    feats = [torch.randn_like(x) for _ in range(4)]
    static = x.clone()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4, capturable=True)
    k = [0]

    def load():
        static.copy_(feats[k[0] % len(feats)])
        k[0] += 1

    def train_body():
        out = call(static).float()
        out.square().mean().backward()
        opt.step()

    def infer_body():
        with torch.no_grad():
            return call(static)

    def eager_train():
        load()
        opt.zero_grad(set_to_none=False)
        train_body()

    def eager_infer():
        load()
        infer_body()

    net.train()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            eager_train()
        net.eval()
        for _ in range(3):
            eager_infer()
    torch.cuda.current_stream().wait_stream(side)
    graphs = {}
    with capture.pinned() as keep:
        net.train()
        opt.zero_grad(set_to_none=False)
        graphs["train"] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs["train"]):
            opt.zero_grad(set_to_none=False)          # grads zeroed inside the graph: each replay is one whole step
            train_body()
        net.eval()
        graphs["infer"] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs["infer"]):
            infer_body()
    arms = {
        "train_eager": (lambda: net.train(), eager_train),
        "train_graph": (lambda: net.train(), lambda: (load(), graphs["train"].replay())),
        "infer_eager": (lambda: net.eval(), eager_infer),
        "infer_graph": (lambda: net.eval(), lambda: (load(), graphs["infer"].replay())),
    }
    times = {a: [] for a in arms}
    for a, (mode, fn) in arms.items():                        # warm every arm
        mode()
        timed(fn, 3)
    for _ in range(rounds):                                    # alternated rounds
        for a, (mode, fn) in arms.items():
            mode()
            times[a].append(timed(fn, steps))
    med = {a: sorted(t)[len(t) // 2] for a, t in times.items()}
    summary = {"shape": name, "rows": int(x.numel() // x.size(-1)),
               "train_ms": {"eager": med["train_eager"], "graph": med["train_graph"],
                            "speedup": med["train_eager"] / med["train_graph"]},
               "infer_ms": {"eager": med["infer_eager"], "graph": med["infer_graph"],
                            "speedup": med["infer_eager"] / med["infer_graph"]},
               "all_ms": times, "pinned_objects": len(keep.objects)}
    del graphs, keep, net, opt
    torch.cuda.empty_cache()
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    shapes = [
        ("dense PNALayer x4, multitask shape (B=128, N=32, F=16, towers=2)", dense_multitask),
        ("DGL PNALayer x4 (75 -> 70, towers=5) + sum readout, one ZINC-shaped batch of 128 graphs", dgl_zinc_batch),
        ("PNAConvSimple(128, 128), config 2 (arxiv-shaped)", pyg_config2),
    ]
    for name, make in shapes:
        print(json.dumps(measure(name, make, args.rounds, args.steps)), flush=True)


if __name__ == "__main__":
    main()
