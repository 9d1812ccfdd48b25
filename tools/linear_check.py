"""On-GPU check of pna_linear_fwd (3xTF32 wgmma) against float64 and timing against cuBLAS fp32."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pna_b200 import linear as L
dev = torch.device("cuda:0")
ok = True
for (n, k, o) in [(128, 32, 128), (1000, 96, 64), (5000, 1536, 128), (300, 64, 256), (169343, 1536, 128)]:
    g = torch.Generator().manual_seed(n + k)
    a = torch.randn(n, k, generator=g).to(dev); w = (torch.randn(o, k, generator=g) / k ** 0.5).to(dev); b = torch.randn(o, generator=g).to(dev)
    y = L.linear_tf32x3(a, w, b); torch.cuda.synchronize()
    ref64 = (a.double() @ w.double().t() + b.double())
    ref32 = torch.nn.functional.linear(a, w, b)
    e_k = (y.double() - ref64).abs().max().item(); e_c = (ref32.double() - ref64).abs().max().item()
    d = (y.double() - ref64)
    bias_to_zero = float((d * torch.sign(ref64)).mean())     # < 0: results shrink towards zero (truncating accumulation)
    rms = float(d.pow(2).mean().sqrt()); rms_c = float((ref32.double() - ref64).pow(2).mean().sqrt())
    print(f"   signed bias {bias_to_zero:.2e}  rms err kernel {rms:.2e}  cuBLAS {rms_c:.2e}")
    good = e_k < 3e-5 * max(1.0, ref64.abs().max().item())
    ok &= good
    ts = []
    for fn in (lambda: L.linear_tf32x3(a, w, b), lambda: torch.nn.functional.linear(a, w, b)):
        for _ in range(3): fn()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(10): fn()
        e.record(); torch.cuda.synchronize(); ts.append(s.elapsed_time(e) / 10)
    print(f"n={n} k={k} o={o}: max|err| kernel {e_k:.2e}  cuBLAS fp32 {e_c:.2e}  {'ok' if good else 'MISMATCH'}   {ts[0]:.3f} ms vs cuBLAS {ts[1]:.3f} ms", flush=True)
print("LINEAR ALL OK" if ok else "LINEAR FAILED")
