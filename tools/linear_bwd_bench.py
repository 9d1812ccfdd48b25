"""python tools/linear_bwd_bench.py [--warmup 5] [--reps 20] [--out DIR]

The backward of the first post-aggregation linear on ONE GPU at config 2 (ogbn-arxiv-shaped, N = 169 343, out = 128):
  * plain    a [N, 1536] -> 128               (linear_tf32x3)
  * compact  a [N, 512] x S = 3 scalers -> 128 (linear_scaled_tf32x3, PNAConvSimple's default)
Two versions, alternated call by call with CUDA events around each call (5 warm-up and 20 timed calls per version):
  * kernels  pna_linear_bwd_data + pna_linear_bwd_weight (3xTF32 wgmma), both gradients and each alone, and what the
             layers run (`layers_both`: pna_linear_bwd_data and the library weight gradient);
  * library  the library-GEMM backward the autograd Functions ran before (restated in `library_bwd`), same splits.
For each kernel the achieved TF32 rate (3 products per multiply-add) against the H100 SXM data sheet's 495 TFLOP/s and the
bytes it must move against 3.35 TB/s, and which of the two bounds it; the max error of both versions against float64 in
the measure of DESIGN section 2 (|g - g64| / sum of |products|).
Then one PNAConvSimple training step (forward + backward of x.square().mean(), CSR cached) at config 2, with x requiring
grad (both gradients) and frozen (weight gradient only: a first layer on raw features), each with
  * the layers' backward (this code: tensor-core input gradient, library weight gradient),
  * the library backward inside the same tensor-core forward (the previous code: `library_bwd` patched in),
  * PNA_B200_TENSOR_LINEAR=0 (library forward and backward).
Prints the card, its power limit and max SM clock with the figures; one JSON line per measurement (also DIR/linear_bwd.json)."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import pna_b200  # noqa: E402
from pna_b200 import linear as L, synth  # noqa: E402

A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]
PEAK_TF32, PEAK_HBM = 495e12, 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as exc:  # noqa: BLE001
        q = f"unknown ({exc})"
    return name, q


def library_bwd(gy, a, c, w, need_a=True, need_w=True):
    """The backward of _Linear3xTF32 / _LinearScaled3xTF32 before the tensor-core kernels, verbatim."""
    if c is None:
        ga = gy @ w if need_a else None
        gw = gy.t() @ a if need_w else None
        return ga, gw
    ka = a.size(1)
    ga = torch.zeros_like(a) if need_a else None
    gw = torch.empty_like(w) if need_w else None
    for s in range(c.size(1)):
        cs = c[:, s:s + 1]
        if ga is not None:
            ga.addcmul_(gy @ w[:, s * ka:(s + 1) * ka], cs)
        if gw is not None:
            torch.mm(gy.t(), a * cs, out=gw[:, s * ka:(s + 1) * ka])
    return ga, gw


def alternate(fns, warmup, reps):
    """ms per call of each fn, calls alternated: median and min over `reps` timed calls."""
    for fn in fns:
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    times = [[] for _ in fns]
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in fns]
    for _ in range(reps):
        for k, fn in enumerate(fns):
            ev[k][0].record()
            fn()
            ev[k][1].record()
            torch.cuda.synchronize()
            times[k].append(ev[k][0].elapsed_time(ev[k][1]))
    return [(statistics.median(t), min(t)) for t in times]


def rel_err(g, g64, cond):
    d = (g.double() - g64).abs()
    return float(torch.where(cond > 0, d / cond.clamp(min=1e-300), d * float("inf")).nan_to_num(0.0).max())


def errors(gy, a, c, w):
    """max elementwise |g - g64| / sum|products| of (ga, gw) for the kernels and the library."""
    ka = a.size(1)
    s_n = 1 if c is None else c.size(1)
    new, lib = L.linear_bwd_tf32x3(gy, a, c, w), library_bwd(gy, a, c, w)
    gy64 = gy.double()
    out = {"kernel_ga": 0.0, "library_ga": 0.0, "kernel_gw": 0.0, "library_gw": 0.0}
    ga64 = torch.zeros(a.shape, dtype=torch.float64, device=a.device)
    ga_cond = torch.zeros_like(ga64)
    for s in range(s_n):
        cols = slice(s * ka, (s + 1) * ka)
        ws = w[:, cols].double()
        cs = 1.0 if c is None else c[:, s:s + 1].double()
        ga64 += cs * (gy64 @ ws)
        ga_cond += (cs.abs() if c is not None else 1.0) * (gy64.abs() @ ws.abs())
        a1 = (a if c is None else a * c[:, s:s + 1]).double()
        gw64, gw_cond = gy64.t() @ a1, gy64.abs().t() @ a1.abs()
        del a1
        out["kernel_gw"] = max(out["kernel_gw"], rel_err(new[1][:, cols], gw64, gw_cond))
        out["library_gw"] = max(out["library_gw"], rel_err(lib[1][:, cols], gw64, gw_cond))
    out["kernel_ga"] = rel_err(new[0], ga64, ga_cond)
    out["library_ga"] = rel_err(lib[0], ga64, ga_cond)
    return {k: float(f"{v:.3e}") for k, v in out.items()}


def roofline(ms, flops, nbytes):
    t_tc, t_hbm = flops / PEAK_TF32, nbytes / PEAK_HBM
    return {"ms": round(ms, 4), "tf32_tflops": round(flops / (ms * 1e-3) / 1e12, 1),
            "tf32_share": round(flops / (ms * 1e-3) / PEAK_TF32, 3), "bytes_gb": round(nbytes / 1e9, 3),
            "hbm_tbs": round(nbytes / (ms * 1e-3) / 1e12, 2), "hbm_share": round(nbytes / (ms * 1e-3) / PEAK_HBM, 3),
            "bound": "tensor" if t_tc >= t_hbm else "HBM", "share_of_bound": round(max(t_tc, t_hbm) / (ms * 1e-3), 3)}


def measure_linear(label, n, ka, s, o, warmup, reps):
    dev = torch.device("cuda:0")
    g = torch.Generator(device=dev).manual_seed(1)
    a = torch.randn(n, ka, generator=g, device=dev)
    c = None
    if s:
        c = torch.rand(n, s, generator=g, device=dev) * 3
        c[:, 0] = 1.0
    k = (s or 1) * ka
    w = torch.randn(o, k, generator=g, device=dev) / k ** 0.5
    gy = torch.randn(n, o, generator=g, device=dev)
    res = {"shape": label, "n_rows": n, "n_in": k, "n_a": ka, "n_scalers": s or 1, "n_out": o}
    fns = {
        "both": (lambda: L.linear_bwd_tf32x3(gy, a, c, w), lambda: library_bwd(gy, a, c, w)),
        # what the autograd Functions run: the tensor-core input gradient and the library weight gradient
        "layers_both": (lambda: (L.linear_bwd_tf32x3(gy, a, c, w, need_w=False), L.library_grad_weight(gy, a, c, w)),
                        lambda: library_bwd(gy, a, c, w)),
        "grad_a": (lambda: L.linear_bwd_tf32x3(gy, a, c, w, need_w=False), lambda: library_bwd(gy, a, c, w, need_w=False)),
        "grad_w": (lambda: L.linear_bwd_tf32x3(gy, a, c, w, need_a=False), lambda: library_bwd(gy, a, c, w, need_a=False)),
    }
    flops = 2.0 * n * o * k * 3                                      # per gradient, 3 tf32 products per multiply-add
    sc = n * (s or 1) * 4 if s else 0
    nbytes = {"grad_a": n * o * 4 + n * ka * 4 + sc, "grad_w": n * o * 4 + n * ka * 4 + sc + o * k * 4}
    for what, (new, lib) in fns.items():
        (m_new, lo_new), (m_lib, lo_lib) = alternate([new, lib], warmup, reps)
        res[f"{what}_kernel_ms"] = round(m_new, 4)
        res[f"{what}_library_ms"] = round(m_lib, 4)
        res[f"{what}_kernel_min_ms"] = round(lo_new, 4)
        res[f"{what}_library_min_ms"] = round(lo_lib, 4)
        res[f"{what}_speedup"] = round(m_lib / m_new, 2)
        if what in nbytes:
            res[f"{what}_roofline"] = roofline(m_new, flops, nbytes[what])
    res["max_rel_err"] = errors(gy, a, c, w)
    return res


def measure_step(warmup, reps):
    dev = torch.device("cuda:0")
    ei, x = synth.arxiv_like(n_feat=128, seed=0)
    n = x.size(0)
    deg = synth.degree_histogram(ei[1], n)
    torch.manual_seed(0)
    lay = pna_b200.PNAConvSimple(128, 128, A4, S3, deg).to(dev)
    eid, xd = ei.to(dev), x.to(dev)
    csr = pna_b200.build_csr(eid[0], eid[1], n)
    assert lay._compact(xd)

    def make_step(x_grad):
        def step():
            xg = xd.detach().requires_grad_(x_grad)
            lay.zero_grad(set_to_none=True)
            lay(xg, eid, csr=csr).square().mean().backward()
        return step

    def with_env(fn, **env):
        def run():
            old = {k: os.environ.get(k) for k in env}
            os.environ.update(env)
            try:
                fn()
            finally:
                for k, v in old.items():
                    if v is None:
                        os.environ.pop(k, None)
                    else:
                        os.environ[k] = v
        return run

    new_bwd = (L._Linear3xTF32.backward, L._LinearScaled3xTF32.backward)

    def old_plain(ctx, gy):
        a, weight = ctx.saved_tensors
        ga, gw = library_bwd(gy, a, None, weight, ctx.needs_input_grad[0], ctx.needs_input_grad[1])
        return ga, gw, gy.sum(0) if (ctx.has_bias and ctx.needs_input_grad[2]) else None

    def old_scaled(ctx, gy):
        a, row_scale, weight = ctx.saved_tensors
        ga, gw = library_bwd(gy, a, row_scale, weight, ctx.needs_input_grad[0], ctx.needs_input_grad[2])
        return ga, None, gw, gy.sum(0) if (ctx.has_bias and ctx.needs_input_grad[3]) else None

    def library_inside(step):
        def run():
            L._Linear3xTF32.backward, L._LinearScaled3xTF32.backward = staticmethod(old_plain), staticmethod(old_scaled)
            try:
                step()
            finally:
                L._Linear3xTF32.backward, L._LinearScaled3xTF32.backward = (staticmethod(new_bwd[0]), staticmethod(new_bwd[1]))
        return run

    res = []
    for x_grad, what in ((True, "x requires grad"), (False, "x frozen: weight gradient only")):
        step = make_step(x_grad)
        (m_new, _), (m_old, _), (m_lib, _) = alternate([step, library_inside(step), with_env(step, PNA_B200_TENSOR_LINEAR="0")],
                                                        warmup, reps)
        res.append({"shape": f"PNAConvSimple training step, config 2 (F = 128, A = 4, S = 3, out 128, CSR cached), {what}",
                    "layers_backward_ms": round(m_new, 3), "library_backward_ms": round(m_old, 3),
                    "tensor_linear_off_ms": round(m_lib, 3), "step_speedup_vs_library_backward": round(m_old / m_new, 3)})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--n", type=int, default=synth.ARXIV_NODES)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("linear_bwd_bench needs a CUDA device")
    name, query = card()
    print(f"card: {name}; nvidia-smi name, power.limit, clocks.max.sm: {query}", flush=True)
    lines = [measure_linear(f"plain [{a.n}, 1536] -> 128", a.n, 1536, 0, 128, a.warmup, a.reps),
             measure_linear(f"compact [{a.n}, 512] x 3 -> 128", a.n, 512, 3, 128, a.warmup, a.reps)]
    torch.cuda.empty_cache()
    lines += measure_step(a.warmup, a.reps)
    for res in lines:
        res.update({"gpu": name, "nvidia_smi": query})
        print(json.dumps(res), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "linear_bwd.json"), "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
