"""python tools/peer_grad_bench.py [--world 8] [--scale 16] [--feat 256] [--out DIR]

The peer plane's backward next to the pull plane's on the same graph, ONE GPU, W ranks in one process (pointers only, as in
tests/test_gpu_peer_grad.py): a config-5-shaped share (10 M nodes, 100 M edges, F = 256 over `world` ranks, 87.5 % of the
edges remote; dist.rank_graph) divided by `scale` so that every rank's buffers fit on one card.  Reports, for rank 0 of
each plane:
  * forward (no gradient) and forward + backward of one differentiable aggregation, the backward as their difference;
  * the peer plane's two backward steps alone: the per-slot kernel (pna_aggregate_bwd_peer_slots) and the return
    (pna_halo_grad_pull over the reverse slot plan), CUDA events after warm-up;
  * what each plane keeps per layer for the backward (pull: the [x ; halo] copy; peer: the ring slot).
All peers' buffers are in this GPU's HBM, so these are local-memory figures, not NVLink ones; the other ranks' buffers hold
random rows (rank 0's timing does not depend on their values).  Prints one JSON line, also written to
DIR/peer_grad_bench.json with --out."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import _lib, dist as pd  # noqa: E402

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


def pools_alloc(world, dev):
    """rank 0's view of every rank's buffers: the i-th allocation of every rank is one random tensor of that shape."""
    pools, calls = {}, {"i": 0}

    def alloc(shape, dt):
        i = calls["i"]
        calls["i"] += 1
        if dt == torch.int64:
            pools[i] = [torch.zeros(shape, dtype=dt, device=dev) for _ in range(world)]
        else:
            pools[i] = [torch.randn(shape, device=dev).to(dt) for _ in range(world)]
        return pools[i][0], [t.data_ptr() for t in pools[i]], None
    return alloc


def fwd_bwd_times(agg_fn, x, gout, warmup, reps):
    with torch.no_grad():
        t_fwd = time_ms(lambda: agg_fn(x), warmup, reps)
    xr = x.clone().requires_grad_(True)

    def fb():
        agg_fn(xr).backward(gout)
        xr.grad = None
    return t_fwd, time_ms(fb, warmup, reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--world", type=int, default=8)
    ap.add_argument("--scale", type=int, default=16)
    ap.add_argument("--feat", type=int, default=256)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("peer_grad_bench needs a CUDA device")
    dev = torch.device("cuda:0")
    W, F = a.world, a.feat
    n_local = 10_000_000 // W // a.scale
    e_local = 100_000_000 // W // a.scale
    bounds = torch.arange(W + 1, dtype=torch.int64) * n_local
    shift = pd.peer_shift_for(bounds)
    edges, plans, cols = [], [], []
    for r in range(W):
        src, dst, _ = pd.rank_graph(r, W, n_local, e_local, 1, p_remote=min(1.0, 0.875 * W / (W - 1)) if W > 1 else 0.0, seed=5)
        edges.append((src, dst))
        plans.append(pd.build_pull_plan(src.to(dev), dst.to(dev), bounds, r, W))
        enc = pd.encode_peer_sources(src.to(dev), bounds, shift)
        cols.append(pna_b200.build_csr(enc, dst.to(dev) - int(bounds[r]), n_local, n_src=W << shift).col)
    src0, dst0 = edges[0]
    deg = torch.bincount(dst0 - int(bounds[0]), minlength=n_local)
    avg = pna_b200.avg_deg_from_histogram(torch.bincount(deg))
    x = torch.randn((n_local, F), device=dev)
    gout = torch.randn((n_local, len(A4) * len(S3) * F), device=dev)
    res = {"what": "peer- and pull-plane backward, rank 0 of an in-process world (local HBM, not NVLink)",
           "world": W, "n_local": n_local, "e_local": e_local, "n_feat": F}

    # pull plane
    pull = pd.PullAggregator(plans[0], F, buffers=2, _alloc=pools_alloc(W, dev), trainable=True,
                             grad_plan=pd.grad_return_plans(plans)[0])
    t_fwd, t_fb = fwd_bwd_times(lambda t: pull.pna_aggregate(t, A4, S3, avg), x, gout, a.warmup, a.reps)
    res.update({"pull_forward_ms": round(t_fwd, 3), "pull_backward_ms": round(t_fb - t_fwd, 3), "pull_n_halo": plans[0].n_halo,
                "pull_saved_bytes_per_layer": (n_local + plans[0].n_halo) * F * 4})
    del pull
    torch.cuda.empty_cache()

    # peer plane
    gplan = pd.peer_grad_return_plans(cols, shift)[0]
    peer = pd.PeerAggregator(src0.to(dev), dst0.to(dev), bounds, 0, W, F, trainable=True, saved_layers=2, grad_plan=gplan,
                             _alloc=pools_alloc(W, dev), _barrier=lambda: None)
    t_fwd, t_fb = fwd_bwd_times(lambda t: peer.pna_aggregate(t, A4, S3, avg), x, gout, a.warmup, a.reps)
    # the two backward steps alone, on the full feature width (one slab at this size)
    csr, L = peer.csr, _lib.lib()
    with torch.no_grad():
        peer.pna_aggregate(x, A4, S3, avg)
    slot = (peer._next - 1) % len(peer._ring)
    st = torch.cuda.current_stream(dev).cuda_stream
    na, ac = _lib.pack_codes(A4, _lib.AGGR_CODES, "aggregator")
    ns, sc = _lib.pack_codes(S3, _lib.SCALER_CODES, "scaler")
    scratch = torch.empty(((csr.n_chunks + csr.n_hubs) * 6, F), device=dev) if csr.n_hubs else None
    d = _lib.AggStruct(gathered=peer._ring[slot].data_ptr(), ld_gathered=F, rowptr=csr.rowptr.data_ptr(), col=csr.col.data_ptr(),
                       n_rows=n_local, n_feat=F, n_towers=1, dtype=_lib.PNA_F32, n_aggr=na, aggr_codes=ac, n_scalers=ns,
                       scaler_codes=sc, avg_log=float(avg["log"]), avg_lin=float(avg["lin"]),
                       split_threshold=csr.split_threshold, chunk_edges=csr.chunk_edges,
                       hub_info=csr.hub_info.data_ptr() if csr.n_hubs else None,
                       chunk_items=csr.chunk_items.data_ptr() if csr.n_hubs else None, n_hubs=csr.n_hubs, n_chunks=csr.n_chunks,
                       hub_partials=None if scratch is None else scratch.data_ptr(),
                       peer_gathered=peer._ring_tables[slot].data_ptr(), peer_shift=shift)
    fc = min(peer._slab, F)
    gs = peer._gbufs[0].view(-1)[: peer._e_max * fc].view(peer._e_max, fc)
    g = torch.zeros((n_local, F), device=dev)
    t_slots = time_ms(lambda: _lib.check(L.pna_aggregate_bwd_peer_slots(C.byref(d), gout.data_ptr(), gout.stride(0), 0, fc,
                                                                        gs.data_ptr(), fc, None, 0, st)), a.warmup, a.reps)
    t_ret = time_ms(lambda: _lib.check(L.pna_halo_grad_pull(peer._gtables[0].data_ptr(), fc, gplan.rows.data_ptr(),
                                                            gplan.rowptr.data_ptr(), gplan.enc.data_ptr(), gplan.shift,
                                                            gplan.n_rows, g.data_ptr(), F, fc, st)), a.warmup, a.reps)
    name, limit = card()
    res.update({"peer_forward_ms": round(t_fwd, 3), "peer_backward_ms": round(t_fb - t_fwd, 3),
                "peer_bwd_slots_ms": round(t_slots, 3), "peer_grad_return_ms": round(t_ret, 3), "peer_slab": peer._slab,
                "peer_slots": csr.n_edges, "peer_return_rows": gplan.n_rows,
                "peer_saved_bytes_per_layer": n_local * F * 4, "peer_slot_buffer_bytes": 2 * peer._e_max * peer._slab * 4,
                "gpu": name, "power_limit": limit})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "peer_grad_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
