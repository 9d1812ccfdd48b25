"""Shared pieces of bench.py / bench_multi.py: peaks, clock sampling, L2 flush, NUMA binding and the in-run parity check.

The parity check is the ONE place outside tests/ and smoke() where the CPU oracle is executed by the bench, and only as the
checker of the CUDA path's output -- never as the thing measured (the cpu_baseline / --impl reference legs time it, which
is their purpose).  Nothing under pna_b200/ imports this module or oracle/.
"""
from __future__ import annotations

import json
import os
import statistics
import subprocess
import threading
from typing import Callable, Optional

import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
AGGRS = ["mean", "max", "min", "std"]
SCALERS = ["identity", "amplification", "attenuation"]
METRIC = "aggregated edges/sec (PNA layer fwd)"
UNIT = "edges/s"
FALLBACK_HBM_GBS = 3350.0     # H100 SXM data sheet HBM3 bandwidth (700 W card); used when no measured peak is supplied
NVLINK_PEER_GBS = 450.0       # H100 SXM data sheet NVLink 4 bandwidth per direction per GPU (900 GB/s both directions)
L2_NOTE = "flushed between timed steps (512 MiB written, then 512 MiB read so no dirty lines remain)"


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured"
        except Exception:
            pass
    return FALLBACK_HBM_GBS, "fallback"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons sampled DURING the timed region."""
    Q = ("index,clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
         "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int):
        self.index, self.rows, self.proc = index, [], None

    def __enter__(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--query-gpu={self.Q}", "--format=csv,noheader,nounits", "-lms", "50",
                                          "-i", str(self.index)], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None
        return self

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([c.strip() for c in line.split(",")])

    def __exit__(self, *a):
        if self.proc is not None:
            self.proc.terminate()
            try:
                self.proc.wait(timeout=2)
            except Exception:
                self.proc.kill()

    def summary(self):
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[1])); mx.append(float(r[2]))
                for nm, v in zip(names, r[4:8]):
                    if v.lower().startswith("active"):
                        reasons.add(nm)
            except Exception:
                continue
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0}
        return {"sm_mhz": statistics.median(sm), "sm_max_mhz": max(mx), "reasons": sorted(reasons), "samples": len(sm)}


class L2Flush:
    """Evict everything of the previous iteration: write 512 MiB, then READ another 512 MiB so the L2 is left full of CLEAN
    lines -- a write-only flush leaves an L2 full (50 MB on H100) of dirty lines whose write-back would be charged to the
    timed step."""

    def __init__(self, dev):
        self.w = torch.empty(512 << 20, dtype=torch.uint8, device=dev)
        self.r = torch.zeros(128 << 20, dtype=torch.float32, device=dev)

    def __call__(self):
        self.w.zero_()
        self.r.sum()


def timed_steps(step: Callable[[], None], k: int, warm: int, flush: Optional[L2Flush], sync: Optional[Callable[[], None]] = None):
    """W untimed + K timed calls of `step`, each timed by its own CUDA event pair on the current stream, L2 flushed before
    every call.  `sync` (multi-GPU: barrier) brackets the timed region together with torch.cuda.synchronize()."""
    for _ in range(warm):
        if flush: flush()
        step()
    starts = [torch.cuda.Event(enable_timing=True) for _ in range(k)]
    ends = [torch.cuda.Event(enable_timing=True) for _ in range(k)]
    torch.cuda.synchronize()
    if sync: sync(); torch.cuda.synchronize()
    for i in range(k):
        if flush: flush()
        starts[i].record()
        step()
        ends[i].record()
    torch.cuda.synchronize()
    if sync: sync(); torch.cuda.synchronize()
    return [s.elapsed_time(t) for s, t in zip(starts, ends)]


def bind_to_gpu_numa(local_rank: int) -> Optional[int]:
    """Pin this process (and with it the pinned host buffers it allocates afterwards) to the NUMA node the GPU hangs off:
    with 8 ranks copying concurrently, host buffers on the far socket halve the PCIe rate of some ranks and make the
    end-to-end step time erratic.  Best effort; returns the node or None."""
    try:
        bus = subprocess.run(["nvidia-smi", "--query-gpu=pci.bus_id", "--format=csv,noheader", "-i", str(local_rank)],
                             capture_output=True, text=True, timeout=10).stdout.strip().lower()
        if bus.startswith("0000"):
            bus = bus[4:]                                   # sysfs uses a 4-digit domain
        node = int(open(f"/sys/bus/pci/devices/{bus}/numa_node").read().strip())
        if node < 0:
            return None
        cpus = []
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus += list(range(int(a), int(b or a) + 1))
        allowed = os.sched_getaffinity(0)
        cpus = [c for c in cpus if c in allowed]
        if cpus:
            os.sched_setaffinity(0, cpus)
            return node
    except Exception:
        pass
    return None


# ---- in-run parity: sampled destination rows of the CUDA output against the CPU oracle ---------------------------------
def sampled_parity(out: torch.Tensor, rowptr: torch.Tensor, col: torch.Tensor, features_of: Callable[[torch.Tensor], torch.Tensor],
                   avg_deg, split_threshold: int, n_rows_sample: int = 100_000, max_edges: int = 4_000_000,
                   big_row_edges: int = 300_000, big_row_cols: int = 32, aggrs=AGGRS, scalers=SCALERS, seed: int = 7,
                   rows: Optional[torch.Tensor] = None) -> dict:
    """Compare `out[r]` for sampled rows r with the oracle (oracle/pna_oracle.py, the reference's op sequence on CPU).

    rowptr / col: the CSR the kernel ran on (device tensors); col[s] indexes SOME source buffer;
    features_of(idx) -> [len(idx), F] CPU tensor with the TRUE feature rows of those source indices (computed from node
    ids, not read back from the device buffer the kernel gathered from -- so a wrong halo exchange shows up here).
    Rows below the split threshold: fp32 oracle, |d| <= 1e-5 + 1e-5 |want| (bf16: 2^-8, 1e-3).  Split rows: the same formulas
    in float64 (tests/test_gpu_parity.py explains why).  Rows with more than `big_row_edges` in-edges are checked on their
    first `big_row_cols` feature columns only, streamed in float64."""
    from oracle import pna_oracle as O
    n = rowptr.numel() - 1
    dev = out.device
    A, S = len(aggrs), len(scalers)
    F = out.size(1) // (A * S)
    g = torch.Generator().manual_seed(seed)
    if rows is None:
        rows = torch.randperm(n, generator=g)[: min(n_rows_sample, n)]
    rows = torch.sort(rows).values
    rp = rowptr.cpu().long()
    deg = rp[rows + 1] - rp[rows]
    big = deg > big_row_edges
    small_rows, small_deg = rows[~big], deg[~big]
    # keep the sample within max_edges (drop the largest rows last: keep prefix of a random order)
    order = torch.randperm(small_rows.numel(), generator=g)
    csum = torch.cumsum(small_deg[order], 0)
    keep = order[: int((csum <= max_edges).sum())]
    small_rows, small_deg = small_rows[keep], small_deg[keep]
    o2 = torch.sort(small_rows)
    small_rows, small_deg = o2.values, small_deg[o2.indices]
    tol = dict(rtol=1e-5, atol=1e-5) if out.dtype == torch.float32 else dict(rtol=2 ** -8, atol=1e-3)
    res = {"rows": int(small_rows.numel()), "edges": int(small_deg.sum()), "max_err_light": 0.0, "max_err_split_vs_f64": 0.0,
           "max_err_over_tol": 0.0, "split_rows": 0, "big_rows": 0, "ok": True}
    if small_rows.numel():
        starts = rp[small_rows]
        slot = torch.repeat_interleave(starts - torch.cumsum(small_deg, 0) + small_deg, small_deg) + torch.arange(int(small_deg.sum()))
        src = col[slot.to(dev)].cpu().long()
        uniq, inv = torch.unique(src, return_inverse=True)
        xu = features_of(uniq).float()
        dst_rel = torch.repeat_interleave(torch.arange(small_rows.numel()), small_deg)
        got = out[small_rows.to(dev)].float().cpu()
        want = O.pyg_aggregate(xu[inv], dst_rel, small_rows.numel(), aggrs, scalers, avg_deg)
        light = small_deg < split_threshold
        if light.any():
            d = (got[light] - want[light]).abs()
            res["max_err_light"] = float(d.max())
            res["max_err_over_tol"] = max(res["max_err_over_tol"], float((d / (tol["atol"] + tol["rtol"] * want[light].abs())).max()))
            res["ok"] &= bool((d <= tol["atol"] + tol["rtol"] * want[light].abs()).all())
        if (~light).any():
            want64 = O.pyg_aggregate(xu.double()[inv], dst_rel, small_rows.numel(), aggrs, scalers, avg_deg)
            d = (got[~light].double() - want64[~light]).abs()
            res["max_err_split_vs_f64"] = float(d.max())
            res["max_err_over_tol"] = max(res["max_err_over_tol"], float((d / (tol["atol"] + tol["rtol"] * want64[~light].abs())).max()))
            res["split_rows"] = int((~light).sum())
            res["ok"] &= bool((d <= tol["atol"] + tol["rtol"] * want64[~light].abs()).all())
    # very large rows: streamed float64 reduction of the first columns
    for r, dg in zip(rows[big].tolist(), deg[big].tolist()):
        c = min(big_row_cols, F)
        s = torch.zeros(c, dtype=torch.float64); q = torch.zeros(c, dtype=torch.float64)
        mn = torch.full((c,), float("inf"), dtype=torch.float64); mx = -mn
        for e0 in range(int(rp[r]), int(rp[r + 1]), 1 << 20):
            idx = col[e0:min(e0 + (1 << 20), int(rp[r + 1]))].cpu().long()
            uq, iv = torch.unique(idx, return_inverse=True)
            cnt = torch.bincount(iv, minlength=uq.numel()).double()
            xr = features_of(uq)[:, :c].double()
            s += (xr * cnt[:, None]).sum(0); q += (xr * xr * cnt[:, None]).sum(0)
            mn = torch.minimum(mn, xr.min(0).values); mx = torch.maximum(mx, xr.max(0).values)
        mean = s / dg
        std = torch.sqrt(torch.clamp(q / dg - mean * mean, min=0) + 1e-5)
        vals = {"mean": mean, "max": mx, "min": mn, "std": std, "sum": s, "var": q / dg - mean * mean}
        lg = torch.log(torch.tensor(float(dg) + 1.0, dtype=torch.float64))
        fac = {"identity": 1.0, "amplification": float(lg) / avg_deg["log"], "attenuation": avg_deg["log"] / float(lg),
               "linear": dg / avg_deg.get("lin", 1.0), "inverse_linear": avg_deg.get("lin", 1.0) / dg}
        got = out[r].double().cpu().view(S, A, F)[:, :, :c]
        for si, sc in enumerate(scalers):
            for ai, ag in enumerate(aggrs):
                want = vals[ag] * fac[sc]
                d = (got[si, ai] - want).abs()
                res["max_err_split_vs_f64"] = max(res["max_err_split_vs_f64"], float(d.max()))
                res["max_err_over_tol"] = max(res["max_err_over_tol"], float((d / (10 * tol["atol"] + 10 * tol["rtol"] * want.abs())).max()))
                res["ok"] &= bool((d <= 10 * tol["atol"] + 10 * tol["rtol"] * want.abs()).all())
        res["big_rows"] += 1
    return res
