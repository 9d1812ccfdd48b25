"""python tools/halo_grad_bench.py [--world 8] [--scale 16] [--feat 256] [--out DIR]

The pull plane's backward on ONE GPU, W ranks in one process (pointers only, as in tests/test_gpu_halo_grad.py): a
config-5-shaped share (10 M nodes, 100 M edges, F = 256 over `world` ranks, 87.5 % of the edges remote) divided by `scale`
so that every rank's buffers fit on one card.  Reports, for rank 0:
  * pna_halo_grad_pull alone (CUDA events after warm-up) and its bytes/s against the HBM peak of the data sheet;
  * the whole per-rank backward (aggregation backward + stage + gradient return) next to the forward (exchange +
    aggregation).
All peers' buffers are in this GPU's HBM, so these are local-memory figures; NVLink behaviour needs >= 2 GPUs
(tools/dist_check.py).  Prints one JSON line, also written to DIR/halo_grad_bench.json with --out."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import _lib, dist as pd  # noqa: E402
from pna_b200.aggregate import backward_mode  # noqa: E402

A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]
HBM_PEAK = 3.35e12          # H100 SXM data sheet, bytes/s


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--scale", type=int, default=16)
    ap.add_argument("--feat", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("halo_grad_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    W, F = a.world, a.feat
    n_local = 10_000_000 // W // a.scale
    e_local = 100_000_000 // W // a.scale
    dsts = []
    plans = []
    bounds = torch.arange(W + 1, dtype=torch.int64) * n_local
    for r in range(W):
        src, dst, _ = pd.rank_graph(r, W, n_local, e_local, 1, p_remote=min(1.0, 0.875 * W / (W - 1)) if W > 1 else 0.0, seed=5)
        plans.append(pd.build_pull_plan(src.to(dev), dst.to(dev), bounds, r, W))
        dsts.append(dst)
    gplans = pd.grad_return_plans(plans)
    rows = max(p.n_local + p.n_halo for p in plans)
    feat = [[torch.zeros((rows, F), device=dev) for _ in range(W)] for _ in range(2)]
    grad = [[torch.randn((rows, F), device=dev) for _ in range(W)] for _ in range(2)]
    flags = [torch.zeros(W, dtype=torch.int64, device=dev) for _ in range(W)]
    calls = {"i": 0}

    def alloc(shape, dt):           # rank 0's view of every rank's buffers
        i = calls["i"]
        calls["i"] += 1
        pool = feat[i] if i < 2 else (flags if i == 2 else grad[i - 3])
        return pool[0], [t.data_ptr() for t in pool], None
    agg = pd.PullAggregator(plans[0], F, buffers=2, _alloc=alloc, trainable=True, grad_plan=gplans[0])
    gp, p0 = gplans[0], plans[0]
    n_slots = int(gp.rowptr[-1])

    # the gradient-return kernel alone
    g = torch.randn((p0.n_local, F), device=dev)
    table = agg._gtables[0]
    st = torch.cuda.current_stream(dev).cuda_stream

    def pull():
        _lib.check(_lib.lib().pna_halo_grad_pull(table.data_ptr(), F, gp.rows.data_ptr(), gp.rowptr.data_ptr(), gp.enc.data_ptr(),
                                                 gp.shift, gp.n_rows, g.data_ptr(), F, F, st))
    t_pull = time_ms(pull, a.warmup, a.reps * 5)
    moved = n_slots * F * 4 + 2 * gp.n_rows * F * 4 + (gp.n_rows * 2 + n_slots) * 4
    bw = moved / (t_pull * 1e-3)

    # forward (exchange + aggregation) and backward (aggregation backward + stage + gradient return) of rank 0
    deg = torch.bincount(dsts[0] - int(bounds[0]), minlength=n_local)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    x = torch.randn((p0.n_local, F), device=dev)
    gout = torch.randn((p0.n_local, len(A4) * len(S3) * F), device=dev)
    with torch.no_grad():
        t_fwd = time_ms(lambda: agg.pna_aggregate(x, A4, S3, avg), a.warmup, a.reps)
    xr = x.clone().requires_grad_(True)

    def fwd_bwd():
        agg.pna_aggregate(xr, A4, S3, avg).backward(gout)
        xr.grad = None
    t_fb = time_ms(fwd_bwd, a.warmup, a.reps)
    name, limit = card()
    res = {"what": "pull-plane backward, rank 0 of an in-process world (local HBM, not NVLink)",
           "gpu": name, "power_limit": limit, "world": W, "n_local": p0.n_local, "e_local": e_local, "n_feat": F,
           "n_halo": p0.n_halo, "grad_return_rows": gp.n_rows, "grad_return_slots": n_slots,
           "grad_pull_ms": round(t_pull, 4), "grad_pull_bytes": moved, "grad_pull_GBps": round(bw / 1e9, 1),
           "grad_pull_of_hbm_peak": round(bw / HBM_PEAK, 3),
           "forward_ms": round(t_fwd, 3), "backward_ms": round(t_fb - t_fwd, 3), "forward_backward_ms": round(t_fb, 3),
           "grad_pull_share_of_backward": round(t_pull / max(t_fb - t_fwd, 1e-9), 4),
           "backward_mode": backward_mode()}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "halo_grad_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
