"""The Set2Set readout on its kernels against the reference's torch loop (cuDNN LSTM), eager and as CUDA-graph replays.

For each shape, a forward and a training step (forward, backward and a capturable Adam step), each run eagerly and as a
replay of a graph captured with torch.cuda.graph, for the kernel readout (pna_b200.S2SReadout) and for the same module
with its Set2Set replaced by the reference's loop in torch ops around a cuDNN nn.LSTM (same parameters).  Inputs are
copied into the static input before every step in all arms.  Median CUDA-event time per step over alternated rounds.
Before timing, the two readouts' outputs are compared at the timed size.  Prints the card and its power limit, then one
JSON line per shape.

    python tools/set2set_bench.py [--rounds 5] [--steps 20]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pna_b200  # noqa: E402
from pna_b200 import capture, dense  # noqa: E402
from pna_b200.nn_blocks import MLP  # noqa: E402

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


class TorchSet2Set(nn.Module):
    """The reference's Set2Set loop: per step one nn.LSTM call, a bmm, a softmax, a weighted sum and a cat."""

    def __init__(self, nin):
        super().__init__()
        self.nin = nin
        self.lstm = nn.LSTM(2 * nin, nin, batch_first=True)

    def forward(self, x):
        B, N, D = x.shape
        hc = (x.new_zeros(1, B, D), x.new_zeros(1, B, D))
        qs = x.new_zeros(B, 1, 2 * D)
        for _ in range(N):
            q, hc = self.lstm(qs, hc)
            a = torch.softmax(torch.matmul(x, q.transpose(1, 2)), dim=1)
            qs = torch.cat([q, (a * x).sum(1, keepdim=True)], -1)
        return qs.squeeze(1)


def readout(kind, d, out=3):
    ro = pna_b200.S2SReadout(d, d, out, fc_layers=3, final_activation="LeakyReLU")
    if kind == "torch":
        ro.set2set = TorchSet2Set(d)
    return ro


class Multitask(nn.Module):
    """The multitask benchmark's net: four dense PNALayers (2 -> 16, then 16 -> 16; towers=2), skip connections into a
    66-wide node MLP and S2SReadout (reference models/pytorch/gnn_framework.py with skip=True, no GRU)."""

    def __init__(self, kind, f=16, nfeat=2):
        super().__init__()
        avg = {"log": 1.6, "lin": 4.8}
        self.convs = nn.ModuleList([dense.PNALayer(nfeat if k == 0 else f, f, AGGRS, SCALERS, avg, towers=2) for k in range(4)])
        w = nfeat + 4 * f
        self.nodes_read_out = MLP(w, w, 3, 3, mid_activation="LeakyReLU", last_activation="LeakyReLU")
        self.graph_read_out = readout(kind, w)

    def forward(self, x, adj):
        skips = [x]
        for conv in self.convs:
            x = conv(x, adj)
            skips.append(x)
        x = torch.cat(skips, 2)
        return self.nodes_read_out(x), self.graph_read_out(x)


def loss_of(out):
    return sum(o.float().square().mean() for o in out) if isinstance(out, tuple) else out.float().square().mean()


def arm_set(net, x, call, rounds_feats):
    """train / infer closures, eager and replayed, for one net on the static input x."""
    static = x.clone()
    opt = torch.optim.Adam(net.parameters(), lr=1e-4, capturable=True)
    k = [0]

    def load():
        static.copy_(rounds_feats[k[0] % len(rounds_feats)])
        k[0] += 1

    def train_body():
        loss_of(call(static)).backward()
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

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        net.train()
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
            opt.zero_grad(set_to_none=False)
            train_body()
        net.eval()
        graphs["infer"] = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graphs["infer"]):
            infer_body()
    arms = {
        "train_eager": (True, eager_train),
        "train_graph": (True, lambda: (load(), graphs["train"].replay())),
        "infer_eager": (False, eager_infer),
        "infer_graph": (False, lambda: (load(), graphs["infer"].replay())),
    }
    return arms, (graphs, keep, opt)


def measure(name, make, rounds, steps):
    torch.manual_seed(0)
    kern, x, call_k = make("kernel")
    ref, _, call_t = make("torch")
    ref.load_state_dict(kern.state_dict())
    kern.eval(), ref.eval()
    # the two Set2Sets agree at the timed size (compared before the MLP, whose outputs are small at initialisation)
    d = kern.graph_read_out.set2set.nin if isinstance(kern, Multitask) else kern.set2set.nin
    xs = torch.randn(x.size(0), x.size(1), d, device=x.device, generator=torch.Generator(x.device).manual_seed(2))
    with torch.no_grad():
        sk = (kern.graph_read_out if isinstance(kern, Multitask) else kern).set2set(xs)
        st = (ref.graph_read_out if isinstance(ref, Multitask) else ref).set2set(xs)
    diff, scale = (sk - st).abs().max().item(), st.abs().max().item()
    assert diff <= 2e-3 * scale, f"{name}: kernel and torch Set2Set differ by {diff} (max |q*| {scale})"
    feats = [torch.randn_like(x) for _ in range(4)]
    arms, keep = {}, []
    for label, (net, call) in (("kernel", (kern, call_k)), ("torch", (ref, call_t))):
        a, k = arm_set(net, x, call, feats)
        keep.append(k)
        arms.update({f"{label}_{n}": (net, mode, fn) for n, (mode, fn) in a.items()})
    times = {a: [] for a in arms}
    for a, (net, mode, fn) in arms.items():                 # warm every arm
        net.train(mode)
        timed(fn, 3)
    for _ in range(rounds):                                  # alternated rounds
        for a, (net, mode, fn) in arms.items():
            net.train(mode)
            times[a].append(timed(fn, steps))
    med = {a: sorted(t)[len(t) // 2] for a, t in times.items()}
    summary = {"shape": name, "set2set_max_abs_diff": diff, "set2set_max_abs": scale}
    for what in ("train", "infer"):
        for how in ("eager", "graph"):
            k, t = med[f"kernel_{what}_{how}"], med[f"torch_{what}_{how}"]
            summary[f"{what}_{how}_ms"] = {"kernel": round(k, 4), "torch": round(t, 4), "speedup": round(t / k, 2)}
    summary["all_ms"] = times
    del keep, arms
    torch.cuda.empty_cache()
    return summary


def s2s_shape(B, N, D):
    def make(kind):
        net = readout(kind, D).cuda()
        x = torch.randn(B, N, D, generator=torch.Generator().manual_seed(1)).cuda()
        return net, x, net
    return make


def multitask_shape():
    B, N = 128, 32
    g = torch.Generator().manual_seed(3)
    adj = (torch.rand(B, N, N, generator=g) < 0.15).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float().cuda()
    x = torch.randn(B, N, 2, generator=g).cuda()

    def make(kind):
        torch.manual_seed(0)
        net = Multitask(kind).cuda()
        return net, x, lambda xx: net(xx, adj)
    return make


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    shapes = [
        ("S2SReadout(16, 16, 3), B=128 graphs of N=32 nodes", s2s_shape(128, 32, 16)),
        ("S2SReadout(66, 66, 3), B=128, N=32 (the multitask skip width)", s2s_shape(128, 32, 66)),
        ("S2SReadout(16, 16, 3), B=128, N=100 (the extrapolation sets' largest graphs)", s2s_shape(128, 100, 16)),
        ("multitask net: 4 dense PNALayers (F=16) + node MLP + S2SReadout(66), B=128, N=32", multitask_shape()),
    ]
    for name, make in shapes:
        print(json.dumps(measure(name, make, args.rounds, args.steps)), flush=True)


if __name__ == "__main__":
    main()
