"""python tools/edge_msg_bench.py [--warmup 5] [--reps 20] [--rounds 3] [--out DIR]

Fused edge messages (pna_edge_msg_fwd / _bwd) against the torch message path (per-tower gathers, concatenations and the
pretrans Linears, then the padded copy) in the DGL PNALayer and the PyG PNAConv, on ONE GPU, CUDA events after warm-up.
The two paths alternate in one run (``rounds`` times each); the torch path is selected by making the layer's kernel check
answer False.  For every shape the two paths' outputs are compared, and the forward (no grad) and a training step
(forward, backward, Adam) are timed, with max_memory_allocated of each; the kernel path is forced for training steps
below edge_mlp.FUSED_TRAINING_MIN_EDGES, and the path the layer itself picks for a step at that size is reported.  Shapes:
  * DGL PNALayer at the reference README's ZINC configuration (hidden 70, towers 5, divide_input, edge_dim 50, L = 1),
    synth.zinc_like with 128 graphs (a training batch) and the full 12 000;
  * DGL PNALayer at the MNIST configuration (hidden 75, towers 5, divide_input, edge_dim 50), synth.superpixel_like,
    128 graphs;
  * PyG PNAConv(128, 128, towers=4, divide_input=True, edge_dim=16, pre_layers=2) on synth.arxiv_like.
Prints the card and its power limit with the figures, one JSON line per measurement (also DIR/edge_msg_bench.json)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import dgl_layers, edge_mlp, pyg, synth  # noqa: E402
from bwd_bench import card, time_ms  # noqa: E402

A4 = "mean max min std"
S3 = "identity amplification attenuation"


def _dgl_shape(name, ei, x, hidden, edge_dim, dev):
    n = x.size(0)
    g = torch.Generator().manual_seed(1)
    e = torch.randn(ei.size(1), edge_dim, generator=g).to(dev)
    indeg = torch.bincount(ei[1], minlength=n).float()
    avg = {"log": float(torch.log(indeg + 1).mean()), "lin": float(indeg.mean())}
    torch.manual_seed(0)
    lay = pna_b200.PNALayer(hidden, hidden, A4, S3, avg, 0.0, True, True, towers=5, divide_input=True, residual=True,
                            edge_features=True, edge_dim=edge_dim).to(dev)
    graph = pna_b200.Graph(ei[0], ei[1], n).to(dev)
    h = x.to(dev)
    snorm = torch.ones(n, 1, device=dev)
    return dict(name=name, layer=lay, cls=dgl_layers.PNALayer, call=lambda: lay(graph, h, e, snorm), n_nodes=n,
                n_edges=ei.size(1))


def _pyg_shape(dev):
    ei, x = synth.arxiv_like()
    n = x.size(0)
    deg = torch.bincount(torch.bincount(ei[1], minlength=n))
    torch.manual_seed(0)
    conv = pna_b200.PNAConv(128, 128, ["mean", "min", "max", "std"], ["identity", "amplification", "attenuation"], deg,
                            towers=4, divide_input=True, edge_dim=16, pre_layers=2).to(dev)
    ea = torch.randn(ei.size(1), 16, generator=torch.Generator().manual_seed(1)).to(dev)
    eid, xd = ei.to(dev), x.to(dev)
    csr = pna_b200.csr_from_edge_index(eid, n)
    return dict(name="PyG PNAConv(128, 128, towers=4, divide_input, edge_dim=16, pre_layers=2), arxiv_like", layer=conv,
                cls=pyg.PNAConv, call=lambda: conv(xd, eid, ea, csr=csr), n_nodes=n, n_edges=ei.size(1))


def measure(s, warmup, reps, rounds):
    lay, cls, call = s["layer"], s["cls"], s["call"]
    opt = torch.optim.Adam(lay.parameters(), lr=1e-4)
    fused_ok = cls._fused_messages_ok
    state = {k: v.clone() for k, v in lay.state_dict().items()}

    min_edges = edge_mlp.FUSED_TRAINING_MIN_EDGES
    with torch.enable_grad():
        chosen = "fused" if edge_mlp.fused_step_pays(s["n_edges"]) else "torch"

    def select(fused):          # fused: the kernel path also for training steps below the layers' size threshold
        cls._fused_messages_ok = fused_ok if fused else (lambda self, *a: False)
        edge_mlp.FUSED_TRAINING_MIN_EDGES = 0 if fused else min_edges

    def fwd():
        with torch.no_grad():
            call()

    def step():
        opt.zero_grad()
        call().pow(2).mean().backward()
        opt.step()

    out = {}
    try:
        for fused in (True, False):                 # outputs from the same parameters
            select(fused)
            with torch.no_grad():
                out[fused] = call().float()
        diff = float((out[True] - out[False]).abs().max() / out[False].abs().max().clamp(min=1e-30))
        t = {(f, k): [] for f in (True, False) for k in ("fwd", "step")}
        mem = {}
        for _ in range(rounds):
            for fused in (True, False):
                select(fused)
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t[(fused, "fwd")].append(time_ms(fwd, warmup, reps))
                t[(fused, "step")].append(time_ms(step, warmup, reps))
                mem[fused] = torch.cuda.max_memory_allocated()
                lay.load_state_dict(state)
    finally:
        cls._fused_messages_ok = fused_ok
        edge_mlp.FUSED_TRAINING_MIN_EDGES = min_edges
    best = {k: min(v) for k, v in t.items()}
    return {"shape": s["name"], "n_nodes": s["n_nodes"], "n_edges": s["n_edges"],
            "max_rel_diff_fused_vs_torch": diff, "training_step_path_the_layer_picks": chosen,
            "fwd_ms": {"fused": round(best[(True, "fwd")], 3), "torch": round(best[(False, "fwd")], 3)},
            "step_ms": {"fused": round(best[(True, "step")], 3), "torch": round(best[(False, "step")], 3)},
            "fwd_ms_all": {"fused": [round(v, 3) for v in t[(True, "fwd")]], "torch": [round(v, 3) for v in t[(False, "fwd")]]},
            "step_ms_all": {"fused": [round(v, 3) for v in t[(True, "step")]],
                            "torch": [round(v, 3) for v in t[(False, "step")]]},
            "max_memory_allocated_MiB": {"fused": round(mem[True] / 2 ** 20, 1), "torch": round(mem[False] / 2 ** 20, 1)}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("edge_msg_bench needs a CUDA GPU")
    dev = torch.device("cuda:0")
    name, limit = card()
    print(f"# {name}, power limit {limit}")
    shapes = []
    for n_graphs in (128, 12_000):
        ei, x, _ = synth.zinc_like(n_graphs=n_graphs, n_feat=70)
        shapes.append(lambda ei=ei, x=x, n_graphs=n_graphs: _dgl_shape(
            f"DGL PNALayer ZINC README shape (hidden 70, towers 5, edge_dim 50), zinc_like {n_graphs} graphs", ei, x, 70, 50,
            dev))
    ei, x = synth.superpixel_like(n_graphs=128, n_feat=75)
    shapes.append(lambda: _dgl_shape("DGL PNALayer MNIST shape (hidden 75, towers 5, edge_dim 50), superpixel_like 128 graphs",
                                     ei, x, 75, 50, dev))
    shapes.append(lambda: _pyg_shape(dev))
    rows = []
    for make in shapes:
        row = measure(make(), a.warmup, a.reps, a.rounds)
        row.update(card=name, power_limit=limit)
        rows.append(row)
        print(json.dumps(row), flush=True)
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "edge_msg_bench.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
