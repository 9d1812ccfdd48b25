"""torchrun --nproc-per-node N tools/dist_check.py : multi-GPU parity of the peer, halo and pull paths against the oracle,
and of the pull, halo and peer paths' backward (the gradient returned to every rank's rows) against the oracle's autograd."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, torch.distributed as dist
from oracle import pna_oracle as O
from pna_b200 import dist as pd

A4, S3 = ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"]
rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
dist.init_process_group("nccl", device_id=dev)
ok = True
for (n, e, f, hubdeg) in [(4000, 40000, 128, 3000), (3000, 20000, 64, 0), (5000, 30000, 256, 600)]:
    g = torch.Generator().manual_seed(n + f)
    src = torch.randint(0, n, (e,), generator=g); dst = torch.randint(0, int(n * 0.95), (e,), generator=g)
    if hubdeg:
        src = torch.cat([src, torch.randint(0, n, (hubdeg,), generator=g)]); dst = torch.cat([dst, torch.full((hubdeg,), 11)])
    x = torch.randn(n, f, generator=g)
    deg = torch.bincount(dst, minlength=n)
    bounds = pd.partition_bounds(deg, world)
    lo, hi = int(bounds[rank]), int(bounds[rank + 1])
    mine = (dst >= lo) & (dst < hi)
    avg = O.avg_deg_from_histogram(torch.bincount(deg))
    want = O.simple_propagate(x, torch.stack([src, dst]), A4, S3, avg)[lo:hi]
    want64 = O.simple_propagate(x.double(), torch.stack([src, dst]), A4, S3, avg)[lo:hi]
    def check(got, tag):
        global ok
        got = got.cpu()
        light = deg[lo:hi] < 256
        good = torch.allclose(got[light], want[light], rtol=1e-5, atol=1e-5) and torch.allclose(got[~light].double(), want64[~light], rtol=1e-5, atol=1e-5)
        ok &= good
        print(f"rank {rank} n={n} f={f} {tag}: max err {(got - want).abs().max().item():.2e} {'ok' if good else 'MISMATCH'}", flush=True)
    # peer path
    pa = pd.PeerAggregator(src[mine].to(dev), dst[mine].to(dev), bounds, rank, world, f)
    pa.x_local.copy_(x[lo:hi].to(dev)); torch.cuda.synchronize(); pa.barrier()
    check(pa.aggregate(A4, S3, avg), "peer[" + pa._keep["how"][:24] + "]")
    # halo path, overlapped and serial
    plan = pd.build_halo_plan(src[mine].to(dev), dst[mine].to(dev), bounds, rank, world)
    for ov in (True, False):
        ha = pd.HaloAggregator(plan, f, overlap=ov)
        ha.x_local.copy_(x[lo:hi].to(dev))
        check(ha.aggregate(A4, S3, avg), f"halo overlap={ov} n_halo={plan.n_halo} interior={int(plan.interior.sum())}")
    # pull path, forward and backward: the gradient every rank gets back for its rows against the oracle's autograd
    pplan = pd.build_pull_plan(src[mine].to(dev), dst[mine].to(dev), bounds, rank, world)
    pull = pd.PullAggregator(pplan, f, trainable=True)
    w = torch.randn(n, 12 * f, generator=torch.Generator().manual_seed(f))
    xr = x.clone().requires_grad_(True)
    (O.simple_propagate(xr, torch.stack([src, dst]), A4, S3, avg) * w).sum().backward()
    xm = x[lo:hi].to(dev).requires_grad_(True)
    out = pull.pna_aggregate(xm, A4, S3, avg)
    (out * w[lo:hi].to(dev)).sum().backward()
    pull.check()
    check(out.detach(), "pull")
    gw, gg = xr.grad[lo:hi], xm.grad.cpu()
    good = torch.allclose(gg, gw, rtol=1e-3, atol=5e-4)
    ok &= good
    print(f"rank {rank} n={n} f={f} pull backward: max err {(gg - gw).abs().max().item():.2e} "
          f"return rows={pull.grad_plan.n_rows} {'ok' if good else 'MISMATCH'}", flush=True)
    # halo path, forward and backward: the gradient goes back through the transposed NCCL all-to-all
    halo = pd.HaloAggregator(plan, f, trainable=True)
    xh = x[lo:hi].to(dev).requires_grad_(True)
    outh = halo.pna_aggregate(xh, A4, S3, avg)
    (outh * w[lo:hi].to(dev)).sum().backward()
    check(outh.detach(), "halo differentiable")
    gh = xh.grad.cpu()
    good = torch.allclose(gh, gw, rtol=1e-3, atol=5e-4)
    ok &= good
    print(f"rank {rank} n={n} f={f} halo backward: max err {(gh - gw).abs().max().item():.2e} "
          f"return rows={halo.grad_plan.n_rows} {'ok' if good else 'MISMATCH'}", flush=True)
    # peer path, forward and backward: per-slot gradients read over NVLink, pulled back by the sources' owners
    peer = pd.PeerAggregator(src[mine].to(dev), dst[mine].to(dev), bounds, rank, world, f, trainable=True)
    xp = x[lo:hi].to(dev).requires_grad_(True)
    outp = peer.pna_aggregate(xp, A4, S3, avg)
    (outp * w[lo:hi].to(dev)).sum().backward()
    peer.check()
    check(outp.detach(), "peer differentiable")
    gp = xp.grad.cpu()
    good = torch.allclose(gp, gw, rtol=1e-3, atol=5e-4)
    ok &= good
    print(f"rank {rank} n={n} f={f} peer backward: max err {(gp - gw).abs().max().item():.2e} "
          f"return rows={peer.grad_plan.n_rows} {'ok' if good else 'MISMATCH'}", flush=True)
    torch.cuda.synchronize(); dist.barrier(device_ids=[local])
t = torch.tensor([1 if ok else 0], device=dev); dist.all_reduce(t, op=dist.ReduceOp.MIN)
if rank == 0: print("DIST ALL OK" if int(t) else "DIST FAILED")
dist.destroy_process_group()
