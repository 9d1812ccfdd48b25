"""python tools/adj_weight_bench.py [--rounds 7] [--reps 20] [--out DIR]

What a weighted adjacency (pna_aggregate_fwd_weighted / _bwd_weighted) costs on ONE GPU against the 0/1 adjacency with the same
pattern.  CUDA events after warm-up; the two variants alternate round by round and the median over rounds is reported:
  * a four-layer dense multitask stack (models/pytorch/pna/layer.py's signature, B x N x N adjacency, aggregators mean max min
    std, scalers identity amplification attenuation) at B=128 N=32 F=16 towers=2 and at B=32 N=64 F=64 towers=2: forward
    (no grad) and one training step (forward, backward, Adam);
  * aggregate_forward / aggregate_backward (atomic and deterministic) at config 2 (ogbn-arxiv-shaped, F = 128 fp32, bench.py's
    graph) without and with slot_weight (random weights in [0.25, 2]).
Prints the card and its power limit with the figures, one JSON line per measurement (also DIR/adj_weight_bench.json with
--out).  The weighted kernels are not tuned (one thread per row and feature column, two passes over the sources)."""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import aggregate as agg, synth  # noqa: E402
from bwd_bench import card, time_ms  # noqa: E402

A4 = ["mean", "max", "min", "std"]
S3 = ["identity", "amplification", "attenuation"]


def alternate(fns, rounds, reps):
    """{name: median ms} over `rounds` rounds, the variants alternating within each round (each warmed up first)."""
    for fn in fns.values():
        time_ms(fn, 3, 1)
    got = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            got[k].append(time_ms(fn, 1, reps))
    return {k: round(statistics.median(v), 4) for k, v in got.items()}


def dense_stack(B, N, F, rounds, reps):
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    mask = (torch.rand(B, N, N, generator=g) < 0.15).float() * (1 - torch.eye(N))
    mask = ((mask + mask.transpose(1, 2)) > 0).float()
    w = torch.rand(B, N, N, generator=g) * 1.75 + 0.25
    adjs = {"01": mask.to(dev), "weighted": (mask * w).to(dev)}
    h = torch.randn(B, N, F, generator=g).to(dev)
    target = torch.randn(B, N, 1, generator=g).to(dev)
    D = mask.sum(-1)
    avg_d = dict(lin=D.mean().item(), log=torch.log(D + 1).mean().item())
    torch.manual_seed(0)
    layers = torch.nn.ModuleList([pna_b200.dense.PNALayer(F, F, A4, S3, avg_d, towers=2) for _ in range(4)]).to(dev)
    head = torch.nn.Linear(F, 1).to(dev)
    opt = torch.optim.Adam(list(layers.parameters()) + list(head.parameters()), lr=1e-4)

    def fwd(adj):
        def run():
            with torch.no_grad():
                z = h
                for lay in layers:
                    z = torch.relu(lay(z, adj))
        return run

    def train(adj):
        def run():
            z = h
            for lay in layers:
                z = torch.relu(lay(z, adj))
            loss = torch.nn.functional.mse_loss(head(z), target)
            opt.zero_grad()
            loss.backward()
            opt.step()
        return run

    what = f"dense multitask stack (B={B} N={N} F={F}, 4 layers, towers=2, {' '.join(A4)})"
    rows = []
    for kind, make in (("forward", fwd), ("training step", train)):
        t = alternate({k: make(a) for k, a in adjs.items()}, rounds, reps)
        rows.append({"what": f"{what} {kind}", "01_ms": t["01"], "weighted_ms": t["weighted"],
                     "ratio": round(t["weighted"] / t["01"], 3)})
    return rows


def aggregation(rounds, reps):
    dev = torch.device("cuda:0")
    ei, x = synth.arxiv_like()
    x = x.to(dev)
    csr = pna_b200.build_csr(ei[0].to(dev), ei[1].to(dev), x.size(0))
    avg = pna_b200.avg_deg_from_histogram(csr.degree_histogram())
    w = (torch.rand(csr.n_edges, generator=torch.Generator().manual_seed(1)) * 1.75 + 0.25).to(dev)
    gout = torch.randn((csr.n_nodes, len(A4) * len(S3) * x.size(1)), device=dev)
    base = {"what": "aggregation config 2", "aggregators": " ".join(A4), "n_rows": csr.n_nodes, "n_edges": csr.n_edges,
            "n_feat": x.size(1)}
    t = alternate({"plain": lambda: agg.aggregate_forward(x, csr, A4, S3, avg),
                   "weighted": lambda: agg.aggregate_forward(x, csr, A4, S3, avg, slot_weight=w)}, rounds, reps)
    rows = [dict(base, call="aggregate_forward", plain_ms=t["plain"], weighted_ms=t["weighted"])]
    for mode in ("atomic", "deterministic"):
        torch.use_deterministic_algorithms(mode == "deterministic")
        try:
            t = alternate({"plain": lambda: agg.aggregate_backward(gout, x, csr, A4, S3, avg),
                           "weighted": lambda: agg.aggregate_backward(gout, x, csr, A4, S3, avg, slot_weight=w)}, rounds, reps)
        finally:
            torch.use_deterministic_algorithms(False)
        rows.append(dict(base, call=f"aggregate_backward ({mode})", plain_ms=t["plain"], weighted_ms=t["weighted"]))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    rows = dense_stack(128, 32, 16, a.rounds, a.reps) + dense_stack(32, 64, 64, a.rounds, a.reps) + aggregation(a.rounds, a.reps)
    for r in rows:
        r.update(card=name, power_limit=limit)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "adj_weight_bench.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
