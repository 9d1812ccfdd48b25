"""Training steps on shuffled mini-batches: the eager loop (a new Graph per batch) against StaticBatch.copy_ + a replayed
CUDA graph of the whole step (build, forward, masked loss, backward, Adam).

Workloads: four DGL PNALayer(-> 70, towers=5) with edge features, graph norm and batch norm, a mean readout and an MLP
readout, on 128-graph batches drawn without replacement from a shuffled pool:
  zinc        ZINC-shaped molecules (synth.zinc_like, 12 000 graphs), 75 input and 16 edge features;
  superpixel  MNIST-superpixel-shaped kNN graphs (70 nodes, k = 8; synth.superpixel_like), 5 input and 2 edge features.
Per training step: the median over alternated rounds of CUDA-event time, the replay time of StaticBatch.build() alone,
and each arm's peak memory.  The card's name and power limit are read in the same run.

    python tools/static_batch_bench.py [--workload zinc|superpixel|all] [--rounds 5] [--steps 40]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pna_b200  # noqa: E402
from pna_b200 import capture, readout, synth  # noqa: E402

DEV = torch.device("cuda:0")
A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]


class Net(nn.Module):
    def __init__(self, in_dim, edge_dim, avg, hidden=70, layers=4):
        super().__init__()
        self.emb = nn.Linear(in_dim, hidden)
        self.layers = nn.ModuleList([
            pna_b200.PNALayer(hidden, hidden, A4, S3, avg, 0.0, True, True, towers=5, divide_input=True, residual=True,
                              edge_features=True, edge_dim=edge_dim) for _ in range(layers)])
        self.mlp = nn.Sequential(nn.Linear(hidden, hidden // 2), nn.ReLU(), nn.Linear(hidden // 2, hidden // 4), nn.ReLU(),
                                 nn.Linear(hidden // 4, 1))

    def forward(self, g, x, e, snorm):
        h = self.emb(x)
        for lay in self.layers:
            h = lay(g, h, e, snorm)
        g.ndata["h"] = h
        return self.mlp(readout.mean_nodes(g, "h")).squeeze(-1)


def workload(name):
    if name == "zinc":
        ei, x, ng = synth.zinc_like(n_graphs=12_000, n_feat=75, seed=0)
        edge_dim = 16
    else:
        n_graphs = 12_000
        ei, x = synth.superpixel_like(n_graphs=n_graphs, nodes_per_graph=70, k=8, n_feat=5, seed=0)
        ng = torch.repeat_interleave(torch.arange(n_graphs), 70)
        edge_dim = 2
    gen = torch.Generator().manual_seed(1)
    e = torch.randn(ei.size(1), edge_dim, generator=gen)
    y = torch.randn(int(ng.max()) + 1, generator=gen)
    indeg = torch.bincount(ei[1], minlength=x.size(0)).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    G = int(ng.max()) + 1
    sizes = torch.bincount(ng, minlength=G)
    esizes = torch.bincount(ng[ei[1]], minlength=G)
    caps = (int(sizes.sort(descending=True).values[:128].sum()), int(esizes.sort(descending=True).values[:128].sum()), 128)
    perm = torch.randperm(G, generator=gen)
    batches = []
    for k in range(G // 128):
        ids = perm[k * 128:(k + 1) * 128]
        sub, bsz, nid, eid = synth.sub_batch(ei, ng, ids)
        n = int(bsz.sum())
        batches.append(dict(ei=sub.pin_memory(), sizes=bsz.tolist(), x=x[nid].pin_memory(), e=e[eid].pin_memory(),
                            snorm=(1.0 / torch.repeat_interleave(bsz.float(), bsz).sqrt()).view(n, 1).pin_memory(),
                            y=y[ids].pin_memory()))
    return batches, x.size(1), edge_dim, avg, caps


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        return out
    except Exception as ex:      # the GPU name from torch is still reported
        return f"{torch.cuda.get_device_name(0)} (nvidia-smi unavailable: {ex})"


def run(name, rounds, steps):
    batches, in_dim, edge_dim, avg, caps = workload(name)
    torch.manual_seed(0)
    eager_net = Net(in_dim, edge_dim, avg).to(DEV).train()
    static_net = Net(in_dim, edge_dim, avg).to(DEV).train()
    static_net.load_state_dict(eager_net.state_dict())
    opt_e = torch.optim.Adam(eager_net.parameters(), lr=1e-3)
    opt_s = torch.optim.Adam(static_net.parameters(), lr=1e-3, capturable=True)
    sb = pna_b200.StaticBatch(*caps, device=DEV)
    y_s = torch.zeros(sb.max_graphs, device=DEV)

    def eager_step(b):
        g = pna_b200.Graph(b["ei"][0].to(DEV, non_blocking=True), b["ei"][1].to(DEV, non_blocking=True), int(sum(b["sizes"])),
                           batch_num_nodes=b["sizes"])
        out = eager_net(g, b["x"].to(DEV, non_blocking=True), b["e"].to(DEV, non_blocking=True),
                        b["snorm"].to(DEV, non_blocking=True))
        opt_e.zero_grad(set_to_none=True)
        ((out - b["y"].to(DEV, non_blocking=True)) ** 2).mean().backward()
        opt_e.step()

    def copy_in(b):
        sb.copy_(src=b["ei"][0], dst=b["ei"][1], batch_num_nodes=b["sizes"], ndata={"x": b["x"], "snorm": b["snorm"]},
                 edata={"e": b["e"]})
        G = len(b["sizes"])
        y_s[:G].copy_(b["y"], non_blocking=True)
        y_s[G:].zero_()

    def static_body():
        sb.build()
        out = static_net(sb, sb.ndata["x"], sb.edata["e"], sb.ndata["snorm"])
        loss = (((out - y_s) ** 2) * sb.graph_mask).sum() / sb.counts[2].float()
        loss.backward()
        opt_s.step()

    # warm-up: every shape of both arms; the static arm on a side stream before its capture
    for b in batches[:3]:
        eager_step(b)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for b in batches[:3]:
            copy_in(b)
            opt_s.zero_grad(set_to_none=True)
            static_body()
    torch.cuda.current_stream().wait_stream(side)
    sb.check()
    step_graph, build_graph = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    opt_s.zero_grad(set_to_none=True)
    with capture.pinned() as keep:
        with torch.cuda.graph(step_graph):
            static_body()
        with torch.cuda.graph(build_graph):
            sb.build()

    def replay_step(b):
        copy_in(b)
        step_graph.replay()

    def timed(fn, k0):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        ev0.record()
        for i in range(steps):
            fn(batches[(k0 + i) % len(batches)])
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) / steps

    res = {"eager": [], "replay": [], "build_replay": []}
    peak = {}
    for r in range(rounds):
        k0 = 3 + r * steps
        for arm, fn in (("eager", eager_step), ("replay", replay_step)) if r % 2 == 0 else \
                (("replay", replay_step), ("eager", eager_step)):
            torch.cuda.reset_peak_memory_stats()
            res[arm].append(timed(fn, k0))
            peak[arm] = max(peak.get(arm, 0), torch.cuda.max_memory_allocated())
        res["build_replay"].append(timed(lambda b: build_graph.replay(), k0))
    sb.check()
    del keep
    med = {k: statistics.median(v) for k, v in res.items()}
    return {"workload": name, "batch_graphs": 128, "capacities": dict(zip(("nodes", "edges", "graphs"), caps)),
            "eager_ms_per_step": round(med["eager"], 3), "replay_ms_per_step": round(med["replay"], 3),
            "build_replay_ms": round(med["build_replay"], 4), "speedup": round(med["eager"] / med["replay"], 2),
            "rounds_ms": {k: [round(v, 3) for v in vs] for k, vs in res.items()},
            "peak_mem_mib": {k: round(v / 2 ** 20, 1) for k, v in peak.items()}, "steps_per_round": steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="all", choices=["zinc", "superpixel", "all"])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=40)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("static_batch_bench needs a CUDA device")
    info = card()
    for w in (["zinc", "superpixel"] if a.workload == "all" else [a.workload]):
        r = run(w, a.rounds, a.steps)
        r["card"] = info
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
