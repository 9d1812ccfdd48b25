"""python tools/pretrans_bench.py [--warmup 5] [--reps 20] [--out DIR]

What pretrans_layers costs in the dense layer on ONE GPU, CUDA events after warm-up:
  * one training step (forward, backward, Adam) of a four-layer dense stack (tools/moments_bench.py's multitask shape,
    B=128 N=32 F=16 towers=2, and one larger shape, B=32 N=64 F=64 towers=2) with pretrans_layers 1, 2 and 3;
  * pna_edge_mlp_fwd against a torch-ops restatement of the same messages (gather, add, bmm per layer), and the
    kernel's backward against autograd of that restatement, alternated in the same run.
Prints the card and its power limit with the figures, one JSON line per measurement (also DIR/pretrans_bench.json with
--out)."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200.edge_mlp import edge_mlp  # noqa: E402
from bwd_bench import card, time_ms  # noqa: E402

A4 = ["mean", "max", "min", "std"]
S3 = ["identity", "amplification", "attenuation"]
SHAPES = [(128, 32, 16), (32, 64, 64)]        # (B, N, F): the multitask stack, and a wider one


def _adjacency(B, N, dev):
    adj = (torch.rand(B, N, N) < 0.15).float() * (1 - torch.eye(N))
    return ((adj + adj.transpose(1, 2)) > 0).float().to(dev)


def dense_step(warmup, reps):
    dev = torch.device("cuda:0")
    rows = []
    for B, N, F in SHAPES:
        torch.manual_seed(0)
        adj = _adjacency(B, N, dev)
        h = torch.randn(B, N, F, device=dev)
        target = torch.randn(B, N, 1, device=dev)
        avg_d = dict(lin=adj.sum(-1).mean().item(), log=torch.log(adj.sum(-1) + 1).mean().item())
        for L in (1, 2, 3):
            layers = torch.nn.ModuleList([pna_b200.dense.PNALayer(F, F, A4, S3, avg_d, towers=2, pretrans_layers=L)
                                          for _ in range(4)]).to(dev)
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
            rows.append({"what": f"dense training step (B={B} N={N} F={F}, 4 layers, towers=2, {' '.join(A4)})",
                         "pretrans_layers": L, "step_ms": round(time_ms(step, warmup, reps), 3)})
    return rows


def _torch_messages(A, Bm, b1, W, bW, i, j, T, Ft):
    """The same messages with torch ops: gather + add, then one batched matrix product per layer."""
    E = i.numel()
    z = torch.relu(A[i] + Bm[j] + b1)
    for k in range(W.size(0)):
        u = torch.bmm(z.view(E, T, Ft).transpose(0, 1), W[k].transpose(1, 2)).transpose(0, 1).reshape(E, T * Ft) + \
            bW[k].reshape(-1)
        z = u if k == W.size(0) - 1 else torch.relu(u)
    return z


def kernel_vs_torch(warmup, reps):
    dev = torch.device("cuda:0")
    rows = []
    for B, N, F in SHAPES:
        torch.manual_seed(1)
        adj = _adjacency(B, N, dev)
        g = pna_b200.dense.dense_graphs(adj, False)
        csr = g.row
        i, j = csr.dst_of_slot, csr.col.long()
        T, Ft = 2, F // 2
        n = B * N
        for L in (2, 3):
            A = torch.randn(n, T * Ft, device=dev, requires_grad=True)
            Bm = torch.randn(n, T * Ft, device=dev, requires_grad=True)
            b1 = torch.randn(T * Ft, device=dev, requires_grad=True)
            W = (torch.randn(L - 1, T, Ft, Ft, device=dev) / Ft ** 0.5).requires_grad_(True)
            bW = torch.randn(L - 1, T, Ft, device=dev, requires_grad=True)
            gM = torch.randn(csr.n_edges, T * Ft, device=dev)
            with torch.no_grad():
                diff = float((edge_mlp(A, Bm, b1, W, bW, csr, T) - _torch_messages(A, Bm, b1, W, bW, i, j, T, Ft)).abs().max())
            fwd = {"kernel": lambda: edge_mlp(A, Bm, b1, W, bW, csr, T).detach(),
                   "torch": lambda: _torch_messages(A, Bm, b1, W, bW, i, j, T, Ft).detach()}
            fb = {"kernel": lambda: torch.autograd.backward(edge_mlp(A, Bm, b1, W, bW, csr, T), gM),
                  "torch": lambda: torch.autograd.backward(_torch_messages(A, Bm, b1, W, bW, i, j, T, Ft), gM)}
            res = {"what": f"edge messages (B={B} N={N} F_t={Ft} towers=2, E={csr.n_edges})", "pretrans_layers": L,
                   "max_abs_diff_kernel_vs_torch": diff}
            for r in range(2):             # alternate the two implementations
                for name in ("kernel", "torch"):
                    with torch.no_grad():
                        res.setdefault(f"{name}_forward_ms", []).append(round(time_ms(fwd[name], warmup, reps), 4))
                    res.setdefault(f"{name}_forward_backward_ms", []).append(round(time_ms(fb[name], warmup, reps), 4))
            rows.append(res)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, limit = card()
    print(f"card: {name}, power limit {limit}", flush=True)
    rows = kernel_vs_torch(a.warmup, a.reps) + dense_step(a.warmup, a.reps)
    for r in rows:
        r.update(card=name, power_limit=limit)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pretrans_bench.json"), "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
