"""fp32 against bf16 autocast for the tower layers, alternated in one run.

For each shape: the forward (autograd on, as in training) and one training step (forward + backward), median CUDA-event
time over the rounds, and the peak memory of a training step (max_memory_allocated above what was allocated before it),
in fp32 and under torch.autocast("cuda", dtype=torch.bfloat16).  Prints the card and its power limit, then one JSON line
per shape.

    python tools/amp_bench.py [--rounds 5] [--steps 10]
"""
from __future__ import annotations

import argparse
import contextlib
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pna_b200  # noqa: E402
from pna_b200 import synth  # noqa: E402

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


def dgl_zinc(n_graphs=12_000, hidden=70, edge_dim=50):
    """The README's ZINC configuration: PNALayer(70, 70, towers=5, divide_input, residual) with edge features."""
    ei, x, _ = synth.zinc_like(n_graphs=n_graphs, n_feat=hidden)
    n = x.size(0)
    e = torch.randn(ei.size(1), edge_dim, generator=torch.Generator().manual_seed(1)).cuda()
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    torch.manual_seed(0)
    lay = pna_b200.PNALayer(hidden, hidden, AGGRS, SCALERS, avg, 0.0, True, True, towers=5, divide_input=True, residual=True,
                            edge_features=True, edge_dim=edge_dim).cuda()
    graph = pna_b200.Graph(ei[0], ei[1], n).to("cuda")
    snorm = torch.ones(n, 1, device="cuda")
    return (lambda hh: lay(graph, hh, e, snorm)), x.cuda(), lay, n, ei.size(1)


def pyg_arxiv(edge_dim=None, pre_layers=1):
    ei, x = synth.arxiv_like(n_feat=128)
    n = x.size(0)
    deg = synth.degree_histogram(ei[1], n)
    torch.manual_seed(0)
    conv = pna_b200.PNAConv(128, 128, AGGRS, SCALERS, deg, towers=4, divide_input=True, edge_dim=edge_dim,
                            pre_layers=pre_layers).cuda()
    eid = ei.cuda()
    csr = pna_b200.csr_from_edge_index(eid, n)
    ea = torch.randn(ei.size(1), edge_dim, generator=torch.Generator().manual_seed(1)).cuda() if edge_dim else None
    return (lambda xx: conv(xx, eid, ea, csr=csr)), x.cuda(), conv, n, ei.size(1)


def measure(name, make, rounds, steps):
    call, x, mod, n, e = make()
    xg = x.clone().requires_grad_(True)
    modes = {"fp32": contextlib.nullcontext, "bf16_autocast": lambda: torch.autocast("cuda", dtype=torch.bfloat16)}

    def fwd(mode):
        with modes[mode]():
            call(xg)

    def train(mode):
        mod.zero_grad(set_to_none=True)
        xg.grad = None
        with modes[mode]():
            out = call(xg)
        out.float().square().mean().backward()

    res = {m: {"fwd_ms": [], "step_ms": []} for m in modes}
    for m in modes:                                             # warm-up and peak memory of a step
        for _ in range(2):
            train(m)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        train(m)
        torch.cuda.synchronize()
        res[m]["peak_step_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    for _ in range(rounds):                                     # alternating rounds
        for m in modes:
            res[m]["fwd_ms"].append(timed(lambda: fwd(m), steps))
            res[m]["step_ms"].append(timed(lambda: train(m), steps))
    summary = {"shape": name, "n_nodes": n, "n_edges": e}
    for m, r in res.items():
        summary[m] = {"fwd_ms_median": sorted(r["fwd_ms"])[len(r["fwd_ms"]) // 2],
                      "step_ms_median": sorted(r["step_ms"])[len(r["step_ms"]) // 2],
                      "peak_step_mib": round(r["peak_step_mib"], 1), "fwd_ms": r["fwd_ms"], "step_ms": r["step_ms"]}
    del call, x, mod, xg
    torch.cuda.empty_cache()
    return summary


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    shapes = [
        ("DGL PNALayer(70, 70, towers=5, divide_input, residual, edge_dim=50), ZINC-shaped, 12 000 graphs", dgl_zinc),
        ("PNAConv(128, 128, towers=4, divide_input=True), arxiv-shaped", lambda: pyg_arxiv()),
        ("PNAConv(128, 128, towers=4, divide_input=True, edge_dim=16, pre_layers=2), arxiv-shaped",
         lambda: pyg_arxiv(16, 2)),
    ]
    for name, make in shapes:
        print(json.dumps(measure(name, make, args.rounds, args.steps)), flush=True)


if __name__ == "__main__":
    main()
