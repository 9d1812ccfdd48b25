"""Compact tower post path against the materialised one (PNA_B200_COMPACT_POST=0), alternating rounds in one run.

For PNAConv and the DGL PNALayer at the shapes the project trains: forward (autograd on, as in training), training step
(forward + backward) and the peak memory of a training step, per path; then a torch.profiler breakdown (CUDA time per
kernel / op) of one DGL ZINC training step on each path.  Prints the card and its power limit, one JSON line per shape,
and writes the profiles to --out.

    python tools/tower_post_bench.py [--rounds 5] [--steps 10] [--out DIR]
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
from pna_b200 import synth  # noqa: E402

AGGRS = ["mean", "max", "min", "std"]
SCALERS = ["identity", "amplification", "attenuation"]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else torch.cuda.get_device_name(0)


def dgl_case(n_graphs, width, edge_dim=None, superpixel=False):
    if superpixel:
        ei, x = synth.superpixel_like(n_graphs=n_graphs, n_feat=width)[:2]
    else:
        ei, x, _ = synth.zinc_like(n_graphs=n_graphs, n_feat=width)
    n = x.size(0)
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    torch.manual_seed(0)
    lay = pna_b200.PNALayer(width, width, AGGRS, SCALERS, avg, 0.0, True, True, towers=5, divide_input=True).cuda()
    graph = pna_b200.Graph(ei[0], ei[1], n).to("cuda")
    h, snorm = x.cuda(), torch.ones(n, 1, device="cuda")
    return (lambda hh: lay(graph, hh, None, snorm)), h, lay, n, ei.size(1)


def pyg_case(edge_dim=None):
    ei, x = synth.arxiv_like(n_feat=128)
    n = x.size(0)
    deg = synth.degree_histogram(ei[1], n)
    torch.manual_seed(0)
    conv = pna_b200.PNAConv(128, 128, AGGRS, SCALERS, deg, towers=4, divide_input=True, edge_dim=edge_dim).cuda()
    eid = ei.cuda()
    csr = pna_b200.csr_from_edge_index(eid, n)
    ea = torch.randn(ei.size(1), edge_dim, device="cuda") if edge_dim else None
    return (lambda xx: conv(xx, eid, ea, csr=csr)), x.cuda(), conv, n, ei.size(1)


pna_b200.linear.TOWERS_COMPACT_MIN_ROWS = 0      # measure both paths at every size: the row threshold is what this measures


def set_path(compact: bool):
    if compact:
        os.environ.pop("PNA_B200_COMPACT_POST", None)
    else:
        os.environ["PNA_B200_COMPACT_POST"] = "0"


def timed(fn, steps):
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        fn()
    t.record()
    torch.cuda.synchronize()
    return s.elapsed_time(t) / steps


def measure(name, make, rounds, steps):
    call, x, mod, n, e = make()
    xg = x.clone().requires_grad_(True)

    def fwd():
        call(xg)

    def train():
        mod.zero_grad(set_to_none=True)
        xg.grad = None
        call(xg).square().mean().backward()

    res = {k: {"fwd_ms": [], "step_ms": []} for k in ("compact", "materialised")}
    outs = {}
    for path in ("compact", "materialised"):                   # warm-up, parity inputs, peak memory
        set_path(path == "compact")
        for _ in range(2):
            train()
        with torch.no_grad():
            outs[path] = call(x)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        train()
        torch.cuda.synchronize()
        res[path]["peak_step_mib"] = (torch.cuda.max_memory_allocated() - base) / 2 ** 20
    for _ in range(rounds):                                     # alternating rounds
        for path in ("compact", "materialised"):
            set_path(path == "compact")
            res[path]["fwd_ms"].append(timed(fwd, steps))
            res[path]["step_ms"].append(timed(train, steps))
    set_path(True)
    summary = {"shape": name, "n_nodes": n, "n_edges": e,
               "max_abs_diff_out": float((outs["compact"] - outs["materialised"]).abs().max())}
    for path, r in res.items():
        summary[path] = {"fwd_ms_median": sorted(r["fwd_ms"])[len(r["fwd_ms"]) // 2], "fwd_ms": r["fwd_ms"],
                         "step_ms_median": sorted(r["step_ms"])[len(r["step_ms"]) // 2], "step_ms": r["step_ms"],
                         "peak_step_mib": r["peak_step_mib"]}
    del call, x, mod, xg
    torch.cuda.empty_cache()
    return summary


def profile(out_dir):
    from torch.profiler import ProfilerActivity, profile as prof
    call, x, mod, n, e = dgl_case(12_000, 70)
    xg = x.clone().requires_grad_(True)
    tables = {}
    for path in ("materialised", "compact"):
        set_path(path == "compact")
        for _ in range(3):
            mod.zero_grad(set_to_none=True)
            call(xg).square().mean().backward()
        torch.cuda.synchronize()
        with prof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
            mod.zero_grad(set_to_none=True)
            call(xg).square().mean().backward()
            torch.cuda.synchronize()
        tables[path] = p.key_averages().table(sort_by="cuda_time_total", row_limit=30)
        with open(os.path.join(out_dir, f"dgl_zinc_step_{path}.txt"), "w") as f:
            f.write(tables[path])
    set_path(True)
    return tables


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    shapes = [
        ("DGL PNALayer(70, 70, towers=5, divide_input), ZINC-shaped, 128 graphs", lambda: dgl_case(128, 70)),
        ("DGL PNALayer(70, 70, towers=5, divide_input), ZINC-shaped, 12 000 graphs", lambda: dgl_case(12_000, 70)),
        ("DGL PNALayer(100, 100, towers=5, divide_input), MNIST-shaped, 128 superpixel graphs",
         lambda: dgl_case(128, 100, superpixel=True)),
        ("PNAConv(128, 128, towers=4, divide_input=True), arxiv-shaped", lambda: pyg_case()),
        ("PNAConv(128, 128, towers=4, divide_input=True, edge_dim=16), arxiv-shaped", lambda: pyg_case(16)),
    ]
    for name, make in shapes:
        print(json.dumps(measure(name, make, args.rounds, args.steps)), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        for path, table in profile(args.out).items():
            print(f"--- one DGL ZINC training step (12 000 graphs), {path} path ---\n{table}", flush=True)


if __name__ == "__main__":
    main()
