"""python tools/bwd_bench.py [--warmup 5] [--reps 20] [--out DIR]

The aggregation's backward (``aggregate_backward``: gradient w.r.t. the gathered rows and row_bias) in its three modes on
ONE GPU, CUDA events after warm-up:
  * atomic         -- pna_aggregate_bwd, one vector atomic per (edge, feature chunk) (the default);
  * coef           -- PNA_B200_BWD=coef: per-destination coefficient rows summed over the transposed graph;
  * deterministic  -- under torch.use_deterministic_algorithms(True): per-slot gradients (pna_aggregate_bwd_slots) summed
                      over the slot-transposed CSR by the forward kernel, no floating-point atomics.
Two shapes: config 2 (ogbn-arxiv-shaped, F = 128, bench.py's workload) and rank 0's share of config 5 divided by 16
(10 M nodes, 100 M edges, F = 256 over 8 ranks, as tools/halo_grad_bench.py; the rank's local CSR over its own and its
halo rows).  The deterministic mode's extra memory is reported: the [E, slab] fp32 per-slot gradients and the
slot-transposed CSR (built once per graph).  Prints the card and its power limit with the figures, one JSON line per
shape (also written to DIR/bwd_bench.json with --out)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import aggregate as agg, dist as pd, synth  # noqa: E402

A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        limit = f"unknown ({exc})"
    return name, limit


def time_ms(fn, warmup, reps):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def csr_bytes(c) -> int:
    return sum(t.numel() * t.element_size() for t in (c.rowptr, c.col, c.perm, c.hub_info, c.chunk_items, c.light_rowptr,
                                                      c.light_deg, c.light_col, c.part) if t is not None)


def measure(label, csr, x, row_bias, avg, warmup, reps):
    dev = x.device
    F = x.size(1)
    gout = torch.randn((csr.n_nodes, len(A4) * len(S3) * F), device=dev)
    res = {"shape": label, "n_rows": csr.n_nodes, "n_src": x.size(0), "n_edges": csr.n_edges, "n_feat": F,
           "split_rows": csr.n_hubs}

    def bwd():
        agg.aggregate_backward(gout, x, csr, A4, S3, avg, row_bias=row_bias, need_bias_grad=row_bias is not None)
    for mode in ("atomic", "coef", "deterministic"):
        os.environ["PNA_B200_BWD"] = "coef" if mode == "coef" else "atomic"
        torch.use_deterministic_algorithms(mode == "deterministic")
        try:
            assert agg.backward_mode() == mode
            res[f"{mode}_ms"] = round(time_ms(bwd, warmup, reps), 3)
        finally:
            torch.use_deterministic_algorithms(False)
            os.environ.pop("PNA_B200_BWD", None)
    slab = agg.deterministic_slab_width(csr.n_edges, F, 16 // x.element_size())
    res["deterministic_slab"] = slab
    res["deterministic_slot_scratch_bytes"] = csr.n_edges * slab * 4
    res["slot_transposed_csr_bytes"] = csr_bytes(csr.slot_transposed(x.size(0)))
    res["deterministic_over_atomic"] = round(res["deterministic_ms"] / res["atomic_ms"], 3)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bwd_bench needs a CUDA device")
    os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")
    dev = torch.device("cuda:0")
    name, limit = card()
    lines = []

    # config 2: ogbn-arxiv-shaped graph, F = 128, gathered rows x (PNAConvSimple)
    ei, x = synth.arxiv_like()
    csr = pna_b200.build_csr(ei[0].to(dev), ei[1].to(dev), x.size(0))
    avg = pna_b200.avg_deg_from_histogram(synth.degree_histogram(ei[1], x.size(0)))
    lines.append(measure("config 2 (arxiv-like, F=128)", csr, x.to(dev), None, avg, a.warmup, a.reps))
    del csr

    # config 5 / 16, rank 0 of 8: the rank's CSR over [local rows ; halo rows], F = 256, with row_bias (PNAConv affine form)
    W, F, scale = 8, 256, 16
    n_local, e_local = 10_000_000 // W // scale, 100_000_000 // W // scale
    bounds = torch.arange(W + 1, dtype=torch.int64) * n_local
    src, dst, _ = pd.rank_graph(0, W, n_local, e_local, 1, p_remote=min(1.0, 0.875 * W / (W - 1)), seed=5)
    plan = pd.build_pull_plan(src.to(dev), dst.to(dev), bounds, 0, W)
    csr = pna_b200.build_csr(plan.src_ext, plan.dst_local, plan.n_local, n_src=plan.n_local + plan.n_halo)
    deg = torch.bincount(dst - int(bounds[0]), minlength=n_local)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    xe = torch.randn((plan.n_local + plan.n_halo, F), device=dev)
    rb = torch.randn((plan.n_local, F), device=dev)
    lines.append(measure("config 5 / 16, rank 0 of 8 (F=256, row_bias)", csr, xe, rb, avg, a.warmup, a.reps))

    for res in lines:
        res.update({"gpu": name, "power_limit": limit})
        print(json.dumps(res))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bwd_bench.json"), "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
