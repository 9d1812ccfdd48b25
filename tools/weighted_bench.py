"""python tools/weighted_bench.py [--warmup 5] [--reps 20] [--out DIR]

What softmax / softmin / normalised_mean cost on ONE GPU, CUDA events after warm-up:
  * aggregate_forward / aggregate_backward (atomic and deterministic) at config 2 (ogbn-arxiv-shaped, F = 128 fp32,
    bench.py's graph) for "mean max min std", that + "softmax softmin", and that + "normalised_mean" (each added to the
    first list: a call takes at most PNA_MAX_AGGR = 6 aggregators), scalers identity amplification attenuation;
  * one training step (forward, backward, Adam) of a dense multitask layer stack (models/pytorch/pna/layer.py's signature,
    B x N x N adjacency) with each of those lists (identity added to the last).
Prints the card and its power limit with the figures, one JSON line per measurement (also DIR/weighted_bench.json with
--out).  The kernels are not tuned (one thread per row and feature, two passes over the sources, scalar loads)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import aggregate as agg, synth  # noqa: E402
from bwd_bench import card, time_ms  # noqa: E402

A4 = ["mean", "max", "min", "std"]
A6 = A4 + ["softmax", "softmin"]
LISTS = (A4, A6, A4 + ["normalised_mean"])
S3 = ["identity", "amplification", "attenuation"]


def aggregation(warmup, reps):
    dev = torch.device("cuda:0")
    ei, x = synth.arxiv_like()
    x = x.to(dev)
    csr = pna_b200.build_csr(ei[0].to(dev), ei[1].to(dev), x.size(0))
    avg = pna_b200.avg_deg_from_histogram(csr.degree_histogram())
    rows = []
    for aggrs in LISTS:
        res = {"what": "aggregation config 2", "aggregators": " ".join(aggrs), "n_rows": csr.n_nodes, "n_edges": csr.n_edges,
               "n_feat": x.size(1)}
        res["forward_ms"] = round(time_ms(lambda: agg.aggregate_forward(x, csr, aggrs, S3, avg), warmup, reps), 3)
        gout = torch.randn((csr.n_nodes, len(aggrs) * len(S3) * x.size(1)), device=dev)
        for mode in ("atomic", "deterministic"):
            torch.use_deterministic_algorithms(mode == "deterministic")
            try:
                res[f"backward_{mode}_ms"] = round(time_ms(lambda: agg.aggregate_backward(gout, x, csr, aggrs, S3, avg), warmup,
                                                           reps), 3)
            finally:
                torch.use_deterministic_algorithms(False)
        rows.append(res)
    return rows


def dense_step(warmup, reps):
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    B, N, F, L = 128, 32, 16, 4               # multitask_benchmark: batches of small graphs, a stack of layers
    adj = (torch.rand(B, N, N) < 0.15).float() * (1 - torch.eye(N))
    adj = ((adj + adj.transpose(1, 2)) > 0).float().to(dev)
    h = torch.randn(B, N, F, device=dev)
    target = torch.randn(B, N, 1, device=dev)
    avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
    rows = []
    for aggrs in (A4, A6, A4 + ["normalised_mean", "identity"]):
        layers = torch.nn.ModuleList([pna_b200.dense.PNALayer(F, F, aggrs, S3, avg_d, towers=2) for _ in range(L)]).to(dev)
        head = torch.nn.Linear(F, 1).to(dev)
        opt = torch.optim.Adam(list(layers.parameters()) + list(head.parameters()), lr=1e-3)

        def step():
            z = h
            for lay in layers:
                z = torch.relu(lay(z, adj))
            loss = torch.nn.functional.mse_loss(head(z), target)
            opt.zero_grad()
            loss.backward()
            opt.step()
        rows.append({"what": f"dense multitask training step (B={B} N={N} F={F}, {L} layers, towers=2)",
                     "aggregators": " ".join(aggrs), "step_ms": round(time_ms(step, warmup, reps), 3)})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    rows = aggregation(a.warmup, a.reps) + dense_step(a.warmup, a.reps)
    for r in rows:
        r.update(card=name, power_limit=limit)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "weighted_bench.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
