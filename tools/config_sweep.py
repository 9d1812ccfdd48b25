"""Time the aggregation on every BASELINE.json config shape that fits one GPU; parity-check a sample of rows.

    python tools/config_sweep.py [--out sweep.json]
Prints one line per config: N, E, F, dtype, ms, edges/s, B_min GB/s, fraction of the measured HBM peak."""
import argparse, json, os, statistics, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import pna_b200
from pna_b200 import synth
from oracle import pna_oracle as O

A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]
dev = torch.device("cuda:0")
ap = argparse.ArgumentParser(); ap.add_argument("--out", default=None); ap.add_argument("--steps", type=int, default=20)
args = ap.parse_args()
peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
    os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")) else 3350.0
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)


def run(name, ei, x, check_rows=2000):
    n, f = x.shape
    e = ei.size(1)
    avg = pna_b200.avg_deg_from_histogram(synth.degree_histogram(ei[1], n))
    xd = x.to(dev)
    csr = pna_b200.build_csr(ei[0].to(dev), ei[1].to(dev), n)
    out = torch.empty((n, 12 * f), dtype=x.dtype, device=dev)
    ts = []
    for i in range(args.steps + 3):
        flush.zero_()
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); pna_b200.aggregate_forward(xd, csr, A4, S3, avg, out=out); t.record(); torch.cuda.synchronize()
        if i >= 3: ts.append(s.elapsed_time(t))
    ms = statistics.median(ts)
    # parity on the sub-graph induced by the first rows' in-edges (oracle on the full graph would take minutes at config 5)
    rows = min(check_rows, n)
    keep = ei[1] < rows
    sub = ei[:, keep]
    want = O.simple_propagate(x.float(), sub, A4, S3, avg)[:rows]
    got = out[:rows].float().cpu()
    deg = torch.bincount(sub[1], minlength=rows)
    light = deg < csr.split_threshold
    tol = dict(rtol=1e-5, atol=1e-5) if x.dtype == torch.float32 else dict(rtol=2 ** -8, atol=1e-3)
    ok = torch.allclose(got[light], want[light], **tol)
    by = synth.algorithmic_bytes(n, e, f, x.element_size(), 12 * f)
    # backward of the aggregation (pna_aggregate_bwd), same graph, upstream gradient of ones
    go = torch.ones_like(out)
    tb = []
    for i in range(5):
        flush.zero_()
        s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); pna_b200.aggregate.aggregate_backward(go, xd, csr, A4, S3, avg); t.record(); torch.cuda.synchronize()
        if i >= 1: tb.append(s.elapsed_time(t))
    rec = {"config": name, "backward_ms": statistics.median(tb), "n_nodes": n, "n_edges": e, "n_feat": f, "dtype": str(x.dtype).replace("torch.", ""), "ms": ms,
           "edges_per_s": e / ms * 1e3, "b_min_gbs": by["b_min"] / ms / 1e6, "frac_of_measured_peak": by["b_min"] / ms / 1e6 / peak,
           "split_rows": csr.n_hubs, "max_in_degree": csr.max_degree, "parity_first_rows": bool(ok)}
    print(json.dumps(rec), flush=True)
    del xd, out, csr
    torch.cuda.empty_cache()
    return rec

recs = []
ei, x = synth.multitask_like(); recs.append(run("1 multitask 64x1k nodes F=16 fp32", ei, x))
ei, x = synth.arxiv_like(); recs.append(run("2 ogbn-arxiv-shaped F=128 fp32", ei, x))
ei, x = synth.arxiv_like(skew=1.0); recs.append(run("2u ogbn-arxiv-shaped, uniform destinations F=128 fp32", ei, x))
ei, x, _ = synth.zinc_like(dtype=torch.bfloat16); recs.append(run("3 ZINC-like 12k graphs F=75 bf16", ei, x))
ei, x, _ = synth.zinc_like(n_feat=80, dtype=torch.bfloat16); recs.append(run("3p ZINC-like, feature pitch padded to F=80 bf16", ei, x))
ei, x = synth.superpixel_like(); recs.append(run("4 superpixels 15k graphs (one GPU's share) F=64 fp32", ei, x))
ei, x = synth.powerlaw(); recs.append(run("5 power-law 1.25M/12.5M (one GPU's share) F=256 fp32", ei, x))
# layer level on ZINC-like dims: PNAConv(75 -> 75, towers 5) fp32, odd tower width 15 -> padded to 16 inside the layer
ei, x, _ = synth.zinc_like(dtype=torch.float32)
n = x.size(0)
lay = pna_b200.PNAConv(75, 75, A4, S3, synth.degree_histogram(ei[1], n), towers=5, divide_input=True).to(dev)
xd, eid = x.to(dev), ei.to(dev)
csr = pna_b200.build_csr(eid[0], eid[1], n)
with torch.no_grad():
    for _ in range(3): lay(xd, eid, csr=csr)
    s, t = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(20): lay(xd, eid, csr=csr)
    t.record(); torch.cuda.synchronize()
rec = {"config": "3L ZINC-like PNAConv(75,75,towers=5) layer forward fp32, CSR cached", "n_nodes": n, "n_edges": ei.size(1),
       "ms": s.elapsed_time(t) / 20, "edges_per_s": ei.size(1) / (s.elapsed_time(t) / 20) * 1e3}
print(json.dumps(rec), flush=True)
recs.append(rec)
if args.out:
    json.dump(recs, open(args.out, "w"), indent=1)
