"""Destination-partitioned multi-GPU PNA aggregation (BASELINE.json configs[4]; SURVEY.md section 8e).

The reference has no distributed code at all (SURVEY.md section 2, "NCCL / collective call sites: None").  Rows
(destinations) are independent, so the graph is cut into contiguous destination ranges, one per GPU / process.  A rank
owns the features and the output rows of its range and all in-edges of its rows; sources may live on other ranks.
Three ways to reach remote source rows, all behind ``pna_aggregate_fwd``:

* ``pull`` (``PullAggregator``, what ``bench.py --gpus N`` times): the rank's DE-DUPLICATED remote sources are listed once
  per graph, locally (the puller names the rows; no id exchange); per layer a device-side flag barrier
  (``pna_peer_barrier``) and ONE kernel of NVLink peer loads (``pna_halo_pull``) fill the halo tail of the rank's
  ``[local ; halo]`` buffer, and the aggregation gathers from local HBM only.  A remote row crosses NVLink once per layer
  however often it is gathered -- what a power-law graph needs.  Trainable (``trainable=True``): the owners pull the halo
  rows' gradients back the same way (``pna_halo_grad_pull``).
* ``halo`` (``HaloAggregator``; the north star's wording, measured beside pull): the same rows through a pack kernel
  (``pna_gather_rows``) and ONE NCCL all-to-all-v (``torch.distributed.all_to_all_single``); rows whose sources are all
  local can be reduced while the all-to-all is in flight (masked light views).  Needs only a process group, so it also
  runs across nodes and between GPUs that cannot map each other's memory.  Trainable (``trainable=True``): the halo
  rows' gradients go back through the transposed all-to-all and the owners add them with ``pna_halo_grad_pull``.
* ``peer`` (``PeerAggregator``): ``col`` encodes ``owner << shift | row`` and the aggregation kernel gathers remote rows
  straight from the owner's HBM with the same asynchronous copies it uses for local rows -- gather and exchange are ONE
  kernel, no halo buffer at all; every remote EDGE crosses the link (peer lines are not cached in the local L2), so it
  fits graphs whose remote rows are rarely reused.

Host-side planning below is plain torch and runs on CPU tensors too (gloo), which is how tests/test_dist_cpu.py covers
it without GPUs.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import List, Optional

import torch
import torch.distributed as dist

from . import _lib, capture
from .aggregate import _DTYPES, _names, _rows2d, aggregate_forward, deterministic_slab_width, pna_aggregate
from .csr import LightView, build_csr


def _refuse_capture(plane) -> None:
    """The planes wait on their peers (barriers with timeouts, collectives, status read-backs): not capturable."""
    capture.guard(f"{type(plane).__name__} (a multi-GPU plane)", "the multi-GPU planes run eagerly only")


# ---- partitioning ------------------------------------------------------------------------------------------------
def partition_bounds(in_degree: torch.Tensor, world: int, row_cost: int = 12) -> torch.Tensor:
    """Contiguous destination ranges of equal cost (in-edges + row_cost per row), int64 [world+1]."""
    n = in_degree.numel()
    cost = torch.cumsum(in_degree.to(torch.int64) + row_cost, 0)
    total = int(cost[-1]) if n else 0
    targets = torch.arange(1, world, dtype=torch.int64) * total // world
    cuts = torch.searchsorted(cost, targets, right=False) + 1 if n else torch.zeros(world - 1, dtype=torch.int64)
    return torch.cat([torch.zeros(1, dtype=torch.int64), cuts.clamp(max=n), torch.tensor([n], dtype=torch.int64)])


def owner_of(ids: torch.Tensor, bounds: torch.Tensor) -> torch.Tensor:
    return torch.bucketize(ids, bounds[1:].to(ids.device), right=True)


def peer_shift_for(bounds: torch.Tensor) -> int:
    biggest = int((bounds[1:] - bounds[:-1]).max())
    shift = max(1, (max(biggest, 1) - 1).bit_length())
    world = bounds.numel() - 1
    if shift > 30 or (world << shift) >= 2 ** 31:
        raise ValueError("partition too large for the 32-bit owner|row encoding")
    return shift


def encode_peer_sources(src_global: torch.Tensor, bounds: torch.Tensor, shift: int) -> torch.Tensor:
    """Global source id -> owner << shift | row-on-owner."""
    b = bounds.to(src_global.device)
    own = owner_of(src_global, bounds)
    return (own << shift) | (src_global - b[own])


@dataclass
class HaloPlan:
    """What one rank needs to run its rows with a [local ; halo] source buffer."""
    rank: int
    world: int
    lo: int
    hi: int
    n_local: int
    n_halo: int
    src_ext: torch.Tensor          # int64 [E_r] sources remapped to [0, n_local + n_halo)
    dst_local: torch.Tensor        # int64 [E_r]
    halo_ids: torch.Tensor         # int64 [n_halo] global ids, sorted (hence grouped by owner)
    recv_splits: List[int]         # rows received from each rank per exchange
    send_splits: List[int]         # rows sent to each rank per exchange
    send_idx: torch.Tensor         # int32 [sum(send_splits)] local rows to send, grouped by destination rank
    interior: torch.Tensor         # bool [n_local]: every source of the row is local


def build_halo_plan(src_global: torch.Tensor, dst_global: torch.Tensor, bounds: torch.Tensor, rank: int, world: int,
                    group=None) -> HaloPlan:
    """src_global -> dst_global are the in-edges of this rank's rows (dst in [bounds[rank], bounds[rank+1]))."""
    dev = src_global.device
    b = bounds.to(dev)
    lo, hi = int(bounds[rank]), int(bounds[rank + 1])
    n_local = hi - lo
    if src_global.numel() and (int(dst_global.min()) < lo or int(dst_global.max()) >= hi):
        raise ValueError("build_halo_plan: an edge's destination is outside this rank's range")
    dst_local = dst_global - lo
    remote = (src_global < lo) | (src_global >= hi)
    halo_ids = torch.unique(src_global[remote])                                   # sorted
    n_halo = int(halo_ids.numel())
    pos = torch.searchsorted(halo_ids, src_global.clamp(min=0)) if n_halo else torch.zeros_like(src_global)
    src_ext = torch.where(remote, n_local + pos, src_global - lo)
    own = owner_of(halo_ids, bounds)
    recv_counts = torch.bincount(own, minlength=world)
    # tell every owner which of its rows we need: counts first, then the (owner-local) ids
    send_counts = torch.empty_like(recv_counts)
    dist.all_to_all_single(send_counts, recv_counts, group=group)
    want = (halo_ids - b[own]).to(torch.int64)
    send_idx = torch.empty(int(send_counts.sum()), dtype=torch.int64, device=dev)
    dist.all_to_all_single(send_idx, want, output_split_sizes=send_counts.tolist(), input_split_sizes=recv_counts.tolist(),
                           group=group)
    has_remote = torch.zeros(n_local, dtype=torch.bool, device=dev)
    if src_global.numel():
        has_remote.index_put_((dst_local[remote],), torch.ones(1, dtype=torch.bool, device=dev).expand(int(remote.sum())))
    return HaloPlan(rank, world, lo, hi, n_local, n_halo, src_ext, dst_local, halo_ids, recv_counts.tolist(),
                    send_counts.tolist(), send_idx.to(torch.int32), ~has_remote)


# ---- device side ---------------------------------------------------------------------------------------------------
def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """out[i] = src[idx[i]] through the C ABI (pna_gather_rows): packs the all-to-all send buffer."""
    if idx.numel() == 0:
        return out
    dt = {torch.float32: _lib.PNA_F32, torch.bfloat16: _lib.PNA_BF16}[src.dtype]
    with torch.cuda.device(src.device):
        _lib.check(_lib.lib().pna_gather_rows(src.data_ptr(), src.stride(0), idx.data_ptr(), idx.numel(), out.data_ptr(),
                                               out.stride(0), src.size(1), dt, torch.cuda.current_stream(src.device).cuda_stream))
    return out


class _HaloExchange(torch.autograd.Function):
    """x [n_local, F] -> a fresh [n_local + n_halo, F] tensor [x ; halo] (``agg.exchange_features``); the backward returns
    the halo rows' gradients to their owners and gives back the fp32 gradient of x (``agg.return_halo_grad``)."""

    @staticmethod
    def forward(ctx, x, agg):
        ctx.agg, ctx.x_dtype = agg, x.dtype
        return agg.exchange_features(x)

    @staticmethod
    def backward(ctx, grad_ext):
        return ctx.agg.return_halo_grad(grad_ext).to(ctx.x_dtype), None


class _TrainableExchange:
    """The differentiable aggregation shared by the planes with a backward.  A plane provides ``plan`` (n_local),
    ``n_feat``, ``dtype``, ``csr`` over ``[local ; halo]``, ``trainable``, ``exchange_features(x)`` and
    ``return_halo_grad(grad_ext)``."""

    def _check_features(self, x: torch.Tensor) -> None:
        n_local = self.plan.n_local
        if tuple(x.shape) != (n_local, self.n_feat) or x.dtype != self.dtype:
            raise ValueError(f"x must be [{n_local}, {self.n_feat}] {self.dtype}, got {tuple(x.shape)} {x.dtype}")

    def pna_aggregate(self, x: torch.Tensor, aggregators, scalers, avg_deg, *, towers: int = 1,
                      row_bias: Optional[torch.Tensor] = None, self_feat: Optional[torch.Tensor] = None,
                      self_divided: bool = True, zero_isolated: bool = False, relu_var: bool = False,
                      scaler_degree: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Differentiable aggregation of this rank's rows (``pna_b200.pna_aggregate`` on ``[x ; halo]``): x is the rank's
        ``[n_local, F]`` features, ``row_bias`` / ``self_feat`` are per destination and stay local; returns the rank's
        ``[n_local, width]`` output.  Every rank must make the same sequence of calls (each one exchanges the halo in the
        forward and, if a gradient flows, returns it in the backward).  Gradients of parameters that produced ``x`` are
        this rank's partial sums: all-reduce them across ranks before the optimizer step."""
        _refuse_capture(self)
        if x.requires_grad and torch.is_grad_enabled() and not self.trainable:
            raise RuntimeError(f"a gradient through the halo exchange needs {type(self).__name__}(..., trainable=True)")
        x_ext = _HaloExchange.apply(x, self)
        return pna_aggregate(x_ext, self.csr, aggregators, scalers, avg_deg, towers=towers, row_bias=row_bias,
                             self_feat=self_feat, self_divided=self_divided, zero_isolated=zero_isolated, relu_var=relu_var,
                             scaler_degree=scaler_degree)


class HaloAggregator(_TrainableExchange):
    """[local ; halo] path: pack -> one NCCL all-to-all-v -> aggregation, interior rows overlapped with the exchange.

    Training (``trainable=True``; opt-in, a forward-only aggregator allocates and communicates nothing more):
    ``pna_aggregate(x, ...)`` is differentiable in ``x``.  Forward: ``x`` into the head of a fresh ``[n_local + n_halo, F]``
    tensor, pack, one all-to-all into its tail (the interior rows' overlap stays on the forward-only ``aggregate()``,
    since the differentiable aggregation is one ``pna_aggregate`` over all rows).  Backward: the
    transposed all-to-all sends every halo row's fp32 gradient back to its owner (``return_halo_grad``), which adds the
    copies of a row into its own gradient in ascending peer rank with ``pna_halo_grad_pull``, without atomics: the
    gradient return is bit-reproducible.  One fp32 receive buffer serves every layer; its reuse is ordered by the stream.
    Parameter gradients are this rank's partial sums; summing them across ranks (``all_reduce``) is the caller's job.
    ``_all_to_all`` replaces ``torch.distributed.all_to_all_single`` (same signature) in both directions: tests run W
    ranks in one process through it."""

    def __init__(self, plan: HaloPlan, n_feat: int, dtype=torch.float32, group=None, overlap: bool = True,
                 trainable: bool = False, _all_to_all=None):
        dev = plan.src_ext.device
        self.plan, self.group, self.overlap, self.n_feat, self.dtype = plan, group, overlap, n_feat, dtype
        self._all_to_all = _all_to_all or dist.all_to_all_single
        self.csr = build_csr(plan.src_ext, plan.dst_local, plan.n_local, n_src=plan.n_local + plan.n_halo)
        self.x_ext = torch.zeros((plan.n_local + plan.n_halo, n_feat), dtype=dtype, device=dev)
        self.send_buf = torch.empty((int(plan.send_idx.numel()), n_feat), dtype=dtype, device=dev)
        self.comm_stream = torch.cuda.Stream(device=dev)
        self.view_interior: Optional[LightView] = None
        self.view_boundary: Optional[LightView] = None
        if overlap:
            self.view_interior = self.csr.masked_view(plan.interior)
            self.view_boundary = self.csr.masked_view(~plan.interior)
        # gradient return (trainable only): owner-side reverse plan, receive buffer, and per peer the start of its segment
        self.trainable, self.grad_plan = trainable, None
        self._grad_recv: Optional[torch.Tensor] = None
        self._grad_table: Optional[torch.Tensor] = None
        if trainable:
            self.grad_plan = halo_grad_return_plan(plan)
            self._grad_recv = torch.empty((int(plan.send_idx.numel()), n_feat), dtype=torch.float32, device=dev)
            starts, off = [], 0
            for n in plan.send_splits:
                starts.append(self._grad_recv.data_ptr() + off * n_feat * 4)
                off += n
            self._grad_table = torch.tensor(starts, dtype=torch.int64, device=dev)

    @property
    def x_local(self) -> torch.Tensor:
        """The rank's own feature rows: produce the layer input in place here (head of the [local ; halo] buffer)."""
        return self.x_ext[: self.plan.n_local]

    def _exchange_into(self, x_ext: torch.Tensor) -> None:
        _refuse_capture(self)
        p = self.plan
        gather_rows(x_ext[:p.n_local], p.send_idx, self.send_buf)
        self._all_to_all(x_ext[p.n_local:], self.send_buf, output_split_sizes=p.recv_splits,
                         input_split_sizes=p.send_splits, group=self.group)

    def exchange(self) -> None:
        self._exchange_into(self.x_ext)

    # ---- differentiable path (trainable=True) ----
    def exchange_features(self, x: torch.Tensor) -> torch.Tensor:
        """Forward half of the differentiable exchange, without autograd: a fresh ``[n_local + n_halo, F]`` tensor
        ``[x ; halo]``, its tail filled by pack + all-to-all."""
        p = self.plan
        self._check_features(x)
        x_ext = torch.empty((p.n_local + p.n_halo, self.n_feat), dtype=self.dtype, device=x.device)
        x_ext[:p.n_local].copy_(x)
        self._exchange_into(x_ext)
        return x_ext

    def return_halo_grad(self, grad_ext: torch.Tensor) -> torch.Tensor:
        """Backward of the exchange: this rank's fp32 gradient for its halo rows goes back to their owners (the forward
        all-to-all with the split sizes swapped; the halo is grouped by owner, so nothing is packed); returns a fp32 copy of
        ``grad_ext[:n_local]`` plus the gradients every peer returned for copies of this rank's rows
        (``pna_halo_grad_pull``, its pointer table aimed at the peers' segments of the local receive buffer)."""
        _refuse_capture(self)
        p, gp = self.plan, self.grad_plan
        if not self.trainable:
            raise RuntimeError("the gradient return needs HaloAggregator(..., trainable=True)")
        send = grad_ext[p.n_local:p.n_local + p.n_halo].to(torch.float32).contiguous()
        self._all_to_all(self._grad_recv, send, output_split_sizes=p.send_splits, input_split_sizes=p.recv_splits,
                         group=self.group)
        dev = self._grad_recv.device
        g = torch.empty((p.n_local, self.n_feat), dtype=torch.float32, device=dev)
        g.copy_(grad_ext[:p.n_local])
        if gp.n_rows:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().pna_halo_grad_pull(self._grad_table.data_ptr(), self.n_feat, gp.rows.data_ptr(),
                                                         gp.rowptr.data_ptr(), gp.enc.data_ptr(), gp.shift, gp.n_rows, g.data_ptr(),
                                                         self.n_feat, self.n_feat, torch.cuda.current_stream(dev).cuda_stream))
        return g

    def aggregate(self, aggregators, scalers, avg_deg, out: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
        _refuse_capture(self)
        main = torch.cuda.current_stream(self.x_ext.device)
        if not self.overlap:
            self.exchange()
            return aggregate_forward(self.x_ext, self.csr, aggregators, scalers, avg_deg, out=out, **kw)
        self.comm_stream.wait_stream(main)                     # x_local is produced on the main stream
        with torch.cuda.stream(self.comm_stream):
            self.exchange()
        out = aggregate_forward(self.x_ext, self.csr, aggregators, scalers, avg_deg, out=out, view=self.view_interior,
                                skip_hubs=True, **kw)          # rows with local sources only: no dependence on the halo
        main.wait_stream(self.comm_stream)
        return aggregate_forward(self.x_ext, self.csr, aggregators, scalers, avg_deg, out=out, view=self.view_boundary, **kw)


@dataclass
class PullPlan:
    """What one rank needs for the pull plane: computed locally from the rank's own in-edges, no id exchange at all
    (the puller names the rows; the owners do nothing)."""
    rank: int
    world: int
    lo: int
    hi: int
    n_local: int
    n_halo: int
    shift: int
    src_ext: torch.Tensor          # int64 [E_r] sources remapped to [0, n_local + n_halo)
    dst_local: torch.Tensor        # int64 [E_r]
    halo_ids: torch.Tensor         # int64 [n_halo] global ids of the de-duplicated remote sources, sorted (grouped by owner)
    enc: torch.Tensor              # int32 [n_halo] owner << shift | row-on-owner
    n_remote_edges: int


def build_pull_plan(src_global: torch.Tensor, dst_global: torch.Tensor, bounds: torch.Tensor, rank: int, world: int) -> PullPlan:
    dev = src_global.device
    lo, hi = int(bounds[rank]), int(bounds[rank + 1])
    n_local = hi - lo
    if src_global.numel() and (int(dst_global.min()) < lo or int(dst_global.max()) >= hi):
        raise ValueError("build_pull_plan: an edge's destination is outside this rank's range")
    remote = (src_global < lo) | (src_global >= hi)
    halo_ids = torch.unique(src_global[remote])
    n_halo = int(halo_ids.numel())
    pos = torch.searchsorted(halo_ids, src_global) if n_halo else torch.zeros_like(src_global)
    src_ext = torch.where(remote, n_local + pos, src_global - lo)
    shift = peer_shift_for(bounds)
    enc = encode_peer_sources(halo_ids, bounds, shift).to(torch.int32) if n_halo else torch.zeros(0, dtype=torch.int32, device=dev)
    return PullPlan(rank, world, lo, hi, n_local, n_halo, shift, src_ext, dst_global - lo, halo_ids, enc, int(remote.sum()))


# ---- backward of the pull and halo planes: return halo gradients to their owners --------------------------------------
@dataclass
class GradReturnPlan:
    """The owner's side of the backward: which of this rank's rows its peers hold as halo copies, and where their
    gradients arrive.  A compact CSR over the rows that have at least one copy; the slots of a row are in ascending peer
    rank, so ``pna_halo_grad_pull`` adds them in a fixed order."""
    rank: int
    world: int
    shift: int                     # enc = peer << shift | position in that peer's segment
    rows: torch.Tensor             # int32 [n_rows] local rows held by at least one peer, ascending
    rowptr: torch.Tensor           # int32 [n_rows + 1]
    enc: torch.Tensor              # int32 [rowptr[-1]]
    # pull plane only: every rank's n_local, where its halo-gradient rows start in its [local ; halo] buffer.  None in the
    # halo plane's plan (halo_grad_return_plan), whose segments are the peers' parts of the local receive buffer.
    peer_n_local: Optional[List[int]] = None
    # peer plane only (peer_grad_return_plan): every rank's number of CSR slots, which sizes the per-slot gradient buffers
    peer_n_edges: Optional[List[int]] = None

    @property
    def n_rows(self) -> int:
        return int(self.rows.numel())


def grad_return_shift(max_halo: int, world: int) -> int:
    """Bits for a halo position: enough for the largest halo of any rank (not the partition size of peer_shift_for)."""
    shift = max(1, (max(int(max_halo), 1) - 1).bit_length())
    if shift > 30 or (world << shift) >= 2 ** 31:
        raise ValueError(f"halo of {max_halo} rows on {world} ranks is too large for the 32-bit peer|position encoding")
    return shift


def grad_return_plan(rank: int, world: int, held: List[torch.Tensor], offsets: List[int], max_halo: int,
                     peer_n_local: Optional[List[int]] = None, device=None) -> GradReturnPlan:
    """Owner ``rank``'s reverse plan from per-peer lists (pure; no communication).

    held[p]   : int64, this rank's rows (owner-local ids, ascending) that rank p holds in its halo;
    offsets[p]: position of the first of them in p's segment (pull plane: p's halo, whose ids are sorted, hence grouped by
                owner, so this rank's rows are one contiguous segment of it and row held[p][i] sits at offsets[p] + i);
    max_halo  : the largest position + 1 any slot can have -- it sizes the position field of the encoding;
    peer_n_local: every rank's n_local, which only the pull plane reads (``PullAggregator``)."""
    shift = grad_return_shift(max_halo, world)
    if device is None:
        device = held[0].device if held else torch.device("cpu")
    rows_l, enc_l = [], []
    for p in range(world):
        ids = held[p].to(device=device, dtype=torch.int64)
        if ids.numel() == 0:
            continue
        if p == rank:
            raise ValueError("grad_return_plan: a rank cannot hold its own rows in its halo")
        pos = int(offsets[p]) + torch.arange(ids.numel(), dtype=torch.int64, device=device)
        rows_l.append(ids)
        enc_l.append((p << shift) | pos)
    n_local = None if peer_n_local is None else list(map(int, peer_n_local))
    return _reverse_csr(rank, world, shift, rows_l, enc_l, device, peer_n_local=n_local)


def _reverse_csr(rank: int, world: int, shift: int, rows_l: List[torch.Tensor], enc_l: List[torch.Tensor], device,
                 **extra) -> GradReturnPlan:
    """The plan's CSR from per-peer (rows, encoded slots) lists appended in ascending peer rank: rows grouped, each row's
    slots kept in the order they were appended (stable sort)."""
    if not rows_l:
        empty = torch.zeros(0, dtype=torch.int32, device=device)
        return GradReturnPlan(rank, world, shift, empty, torch.zeros(1, dtype=torch.int32, device=device), empty.clone(),
                              **extra)
    rows, enc = torch.cat(rows_l), torch.cat(enc_l)
    order = torch.sort(rows, stable=True).indices          # peers were appended in rank order: stable keeps it per row
    rows, enc = rows[order], enc[order]
    uniq, counts = torch.unique_consecutive(rows, return_counts=True)
    rowptr = torch.zeros(uniq.numel() + 1, dtype=torch.int64, device=device)
    rowptr[1:] = torch.cumsum(counts, 0)
    return GradReturnPlan(rank, world, shift, uniq.to(torch.int32), rowptr.to(torch.int32), enc.to(torch.int32), **extra)


# ---- backward of the peer plane: per-slot gradients pulled by the owners of the source rows ------------------------------
def peer_grad_return_plan(rank: int, world: int, rows: List[torch.Tensor], slots: List[torch.Tensor], n_edges: List[int],
                          device=None) -> GradReturnPlan:
    """Owner ``rank``'s reverse slot plan for the peer plane (pure; no communication).

    rows[p]  : int64, this rank's rows (owner-local ids) that the slots of rank p's CSR gather;
    slots[p] : int64, those slots (ascending), one per entry of rows[p].  The owner's own slots are listed under p = rank;
    n_edges  : every rank's number of CSR slots.  The position field of ``enc = p << shift | slot`` covers the largest.
    Each row's slots come out in ascending (rank, slot) order: the slot order of the whole graph's destination-sorted CSR,
    since the ranks own consecutive destination ranges."""
    shift = grad_return_shift(max(map(int, n_edges), default=0), world)
    if device is None:
        device = rows[0].device if rows else torch.device("cpu")
    rows_l, enc_l = [], []
    for p in range(world):
        ids = rows[p].to(device=device, dtype=torch.int64)
        if ids.numel() == 0:
            continue
        s = slots[p].to(device=device, dtype=torch.int64)
        if s.numel() != ids.numel():
            raise ValueError("peer_grad_return_plan: rows and slots differ in length")
        rows_l.append(ids)
        enc_l.append((p << shift) | s)
    return _reverse_csr(rank, world, shift, rows_l, enc_l, device, peer_n_edges=list(map(int, n_edges)))


def _slots_by_owner(col: torch.Tensor, shift: int, world: int):
    """(owner-local rows, slot ids, slots per owner) of one rank's CSR, grouped by owner, slots ascending within an owner."""
    c = col.to(torch.int64)
    own = c >> shift
    order = torch.sort(own, stable=True).indices
    counts = torch.bincount(own, minlength=world) if c.numel() else torch.zeros(world, dtype=torch.int64, device=c.device)
    return (c & ((1 << shift) - 1))[order], order, counts


def peer_grad_return_plans(cols: List[torch.Tensor], shift: int) -> List[GradReturnPlan]:
    """Every rank's reverse slot plan from every rank's CSR ``col`` (entries ``owner << shift | row``), in one process
    (what build_peer_grad_return_plan computes with collectives)."""
    world = len(cols)
    segs = [_slots_by_owner(c, shift, world) for c in cols]
    n_edges = [int(c.numel()) for c in cols]
    out = []
    for r in range(world):
        rows, slots = [], []
        for p in range(world):
            rw, sl, counts = segs[p]
            o = int(counts[:r].sum())
            c = int(counts[r])
            rows.append(rw[o:o + c])
            slots.append(sl[o:o + c])
        out.append(peer_grad_return_plan(r, world, rows, slots, n_edges, device=cols[r].device))
    return out


def build_peer_grad_return_plan(col: torch.Tensor, shift: int, rank: int, world: int, group=None) -> GradReturnPlan:
    """This rank's reverse slot plan, once per graph, with two collectives: an all-to-all of (slot count, edge count) per
    rank pair, then an all-to-all of the (owner-local row, slot) pairs, each rank's grouped by owner."""
    dev = col.device
    rows, slots, counts = _slots_by_owner(col, shift, world)
    meta = torch.stack([counts, torch.full_like(counts, int(col.numel()))], 1)
    meta_in = torch.empty_like(meta)
    dist.all_to_all_single(meta_in, meta.contiguous(), group=group)
    recv = meta_in[:, 0].tolist()
    pairs = torch.empty((sum(recv), 2), dtype=torch.int64, device=dev)
    dist.all_to_all_single(pairs, torch.stack([rows, slots], 1).contiguous(), output_split_sizes=recv,
                           input_split_sizes=counts.tolist(), group=group)
    got = list(torch.split(pairs, recv))
    return peer_grad_return_plan(rank, world, [t[:, 0] for t in got], [t[:, 1] for t in got], meta_in[:, 1].tolist(),
                                 device=dev)


def halo_grad_return_plan(plan: HaloPlan) -> GradReturnPlan:
    """The halo plane's reverse plan, from the owner's own ``HaloPlan`` (pure, local; no collective).  In the backward,
    peer p returns the gradients of the rows this rank sent it, in the order it sent them: the owner's receive buffer holds
    p's segment at ``send_off[p]``, and position ``send_off[p] + q`` carries the gradient of local row
    ``send_idx[send_off[p] + q]``.  Slot encoding: ``p << shift | q``, q < send_splits[p]."""
    held = list(torch.split(plan.send_idx.to(torch.int64), plan.send_splits))
    return grad_return_plan(plan.rank, plan.world, held, [0] * plan.world, max(plan.send_splits, default=0),
                            device=plan.send_idx.device)


def _halo_segments(plan: PullPlan):
    """(owner-local ids grouped by owner, rows per owner, offset of each owner's segment) of a puller's halo."""
    own = (plan.enc >> plan.shift).to(torch.int64)
    want = (plan.enc & ((1 << plan.shift) - 1)).to(torch.int64)
    counts = torch.bincount(own, minlength=plan.world) if plan.n_halo else torch.zeros(plan.world, dtype=torch.int64,
                                                                                          device=plan.enc.device)
    offsets = torch.cumsum(counts, 0) - counts
    return want, counts, offsets


def grad_return_plans(plans: List[PullPlan]) -> List[GradReturnPlan]:
    """Every rank's reverse plan from every rank's PullPlan, in one process (what build_grad_return_plan computes with
    collectives)."""
    world = len(plans)
    max_halo = max(p.n_halo for p in plans)
    n_local = [p.n_local for p in plans]
    segs = [_halo_segments(p) for p in plans]
    out = []
    for r in range(world):
        held, offs = [], []
        for p in range(world):
            want, counts, offsets = segs[p]
            o, c = int(offsets[r]), int(counts[r])
            held.append(want[o:o + c])
            offs.append(o)
        out.append(grad_return_plan(r, world, held, offs, max_halo, n_local, device=plans[r].enc.device))
    return out


def build_grad_return_plan(plan: PullPlan, group=None) -> GradReturnPlan:
    """This rank's reverse plan, once per graph, with two collectives: an all-to-all of (row count, segment offset,
    n_local, n_halo) per rank pair, then an all-to-all of the owner-local row ids (``build_halo_plan``'s pattern)."""
    dev = plan.enc.device
    world = plan.world
    want, counts, offsets = _halo_segments(plan)
    meta = torch.stack([counts, offsets, torch.full_like(counts, plan.n_local), torch.full_like(counts, plan.n_halo)], 1)
    meta_in = torch.empty_like(meta)
    dist.all_to_all_single(meta_in, meta.contiguous(), group=group)
    recv_counts = meta_in[:, 0].tolist()
    ids = torch.empty(sum(recv_counts), dtype=torch.int64, device=dev)
    dist.all_to_all_single(ids, want, output_split_sizes=recv_counts, input_split_sizes=counts.tolist(), group=group)
    held = list(torch.split(ids, recv_counts))
    return grad_return_plan(plan.rank, world, held, meta_in[:, 1].tolist(), int(meta_in[:, 3].max()), meta_in[:, 2].tolist(),
                            device=dev)


class PullAggregator(_TrainableExchange):
    """[local ; halo] source buffer whose halo tail is filled by ONE kernel of peer loads (``pna_halo_pull``): the
    all-to-all of the north star without a collective -- no id exchange when the graph is planned, no pack kernel, no
    send buffer, no NCCL call per layer; a remote row crosses NVLink once per layer however often it is gathered.

    Protocol (one layer): every rank writes its rows into ``x_local`` -> ``exchange()`` = device-side barrier
    (``pna_peer_barrier``: one flag store per peer, spin on the own flags) + the pull -> aggregation from the local
    buffer.  The feature buffer is DOUBLE-BUFFERED (``flip()`` between layers / steps): a rank may already be writing
    layer l+1's rows while slower peers still pull layer l's, and the barrier of layer l+1 separates layer l's pulls
    from the writes of layer l+2 into the same buffer.

    Training (``trainable=True``; opt-in, a forward-only aggregator allocates and communicates nothing more):
    ``pna_aggregate(x, ...)`` is differentiable in ``x``.  Forward: ``x`` -> ``x_local``, barrier, pull, and a copy of
    ``[x ; halo]`` that the next layers' reuse of the double buffers cannot overwrite (the backward reads it: n_local +
    n_halo rows per layer), then ``flip()``.  Backward: the gradient of the halo rows goes into this rank's fp32 gradient
    buffer (``stage_halo_grad``), then a barrier, then every owner pulls the gradients its peers hold for copies of its
    rows and adds them into its own (``pull_halo_grad``, ``pna_halo_grad_pull``).  The slots of a row are added in
    ascending peer rank, without atomics: the gradient return is bit-reproducible.  The gradient buffers alternate like
    the feature buffers, by the same argument: backward exchange j+2 rewrites the buffer that peers pulled from in
    exchange j only after this rank has passed barrier j+1, which no peer enters before its pull of exchange j is done.
    Parameter gradients are this rank's partial sums; summing them across ranks (``all_reduce``) is the caller's job.
    """

    def __init__(self, plan: PullPlan, n_feat: int, dtype=torch.float32, group=None, buffers: int = 2, _alloc=None,
                 trainable: bool = False, grad_plan: Optional[GradReturnPlan] = None, _barrier=None):
        dev = plan.src_ext.device
        self.plan, self.group, self.n_feat, self.dtype = plan, group, n_feat, dtype
        self.csr = build_csr(plan.src_ext, plan.dst_local, plan.n_local, n_src=plan.n_local + max(plan.n_halo, 0))
        rows = torch.tensor([plan.n_local + plan.n_halo], dtype=torch.int64, device=dev)
        if _alloc is None and plan.world > 1:
            dist.all_reduce(rows, op=dist.ReduceOp.MAX, group=group)
        alloc = _alloc or (lambda shape, dt: _symmetric_tensor(shape, dt, dev, plan.rank, plan.world, group))
        self._bufs, self._tables, self._keep = [], [], []
        for _ in range(buffers):
            t, ptrs, keep = alloc((int(rows), n_feat), dtype)
            self._bufs.append(t)
            self._tables.append(torch.tensor(ptrs, dtype=torch.int64, device=dev))
            self._keep.append(keep)
        flags, fptrs, keep = alloc((max(plan.world, 1),), torch.int64)
        flags.zero_()
        self._flags, self._flag_table = flags, torch.tensor(fptrs, dtype=torch.int64, device=dev)
        self._keep.append(keep)
        self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._epoch, self._cur = 0, 0
        # gradient return (trainable only): fp32 buffers whose halo tails the owners pull from, like the feature buffers
        self.trainable, self.grad_plan = trainable, None
        self._gbufs, self._gtables, self._gcur = [], [], 0
        if trainable:
            if grad_plan is None:
                grad_plan = build_grad_return_plan(plan, group) if plan.world > 1 else grad_return_plan(
                    plan.rank, 1, [torch.zeros(0, dtype=torch.int64, device=dev)], [0], plan.n_halo, [plan.n_local], device=dev)
            if grad_plan.rank != plan.rank or grad_plan.world != plan.world:
                raise ValueError("grad_plan belongs to another rank or world")
            if grad_plan.peer_n_local is None:
                raise ValueError("grad_plan has no peer_n_local: it is not a pull-plane reverse plan")
            self.grad_plan = grad_plan
            for _ in range(buffers):
                t, ptrs, keep = alloc((int(rows), n_feat), torch.float32)
                tails = [int(ptrs[p]) + grad_plan.peer_n_local[p] * n_feat * 4 for p in range(len(ptrs))]
                self._gbufs.append(t)
                self._gtables.append(torch.tensor(tails, dtype=torch.int64, device=dev))
                self._keep.append(keep)
        self._barrier_hook = _barrier      # host-side stand-in for the device barrier (several ranks in one process)
        self.use_barrier = (plan.world > 1 and _alloc is None) or _barrier is not None
        if self.use_barrier and _barrier is None:   # flags are zero everywhere before the first flag store can arrive
            torch.cuda.synchronize(dev)
            dist.barrier(group=group, device_ids=[dev.index])

    @property
    def x_ext(self) -> torch.Tensor:
        return self._bufs[self._cur][: self.plan.n_local + self.plan.n_halo]

    @property
    def x_local(self) -> torch.Tensor:
        """This rank's own feature rows: produce the layer input in place here (head of the [local ; halo] buffer)."""
        return self._bufs[self._cur][: self.plan.n_local]

    def flip(self) -> None:
        self._cur = (self._cur + 1) % len(self._bufs)

    def barrier(self) -> None:
        if self._barrier_hook is not None:
            self._barrier_hook()
            return
        self._epoch += 1
        dev = self._flags.device
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().pna_peer_barrier(self._flag_table.data_ptr(), self.plan.rank, self.plan.world, self._epoch, 0,
                                                   self._status.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))

    def exchange(self) -> None:
        _refuse_capture(self)
        p = self.plan
        if self.use_barrier:
            self.barrier()
        if p.n_halo == 0:
            return
        buf = self._bufs[self._cur]
        dt = {torch.float32: _lib.PNA_F32, torch.bfloat16: _lib.PNA_BF16}[self.dtype]
        dev = buf.device
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().pna_halo_pull(self._tables[self._cur].data_ptr(), buf.stride(0), p.enc.data_ptr(), p.shift, p.n_halo,
                                                buf[p.n_local:].data_ptr(), buf.stride(0), self.n_feat, dt,
                                                torch.cuda.current_stream(dev).cuda_stream))

    def aggregate(self, aggregators, scalers, avg_deg, out: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
        self.exchange()
        return aggregate_forward(self.x_ext, self.csr, aggregators, scalers, avg_deg, out=out, **kw)

    # ---- differentiable path (trainable=True) ----
    def exchange_features(self, x: torch.Tensor) -> torch.Tensor:
        """Forward half of the differentiable exchange, without autograd: ``x`` -> ``x_local``, barrier, pull; returns a
        fresh ``[n_local + n_halo, F]`` copy of ``[x ; halo]`` and flips to the other feature buffer."""
        self._check_features(x)
        self.x_local.copy_(x)
        self.exchange()
        out = self.x_ext.clone()
        self.flip()
        return out

    def stage_halo_grad(self, grad_ext: torch.Tensor) -> None:
        """Backward, first half: this rank's gradient for its halo rows -> the halo tail of its current fp32 gradient
        buffer, where the rows' owners pull it from."""
        p = self.plan
        if not self.trainable:
            raise RuntimeError("the gradient return needs PullAggregator(..., trainable=True)")
        if p.n_halo:
            self._gbufs[self._gcur][p.n_local:p.n_local + p.n_halo].copy_(grad_ext[p.n_local:p.n_local + p.n_halo])

    def pull_halo_grad(self, grad_ext: torch.Tensor) -> torch.Tensor:
        """Backward, second half: barrier, then a fp32 copy of ``grad_ext[:n_local]`` plus the gradients every peer staged
        for copies of this rank's rows (``pna_halo_grad_pull``); flips to the other gradient buffer."""
        _refuse_capture(self)
        p, gp = self.plan, self.grad_plan
        if not self.trainable:
            raise RuntimeError("the gradient return needs PullAggregator(..., trainable=True)")
        if self.use_barrier:
            self.barrier()
        dev = self._gbufs[self._gcur].device
        g = torch.empty((p.n_local, self.n_feat), dtype=torch.float32, device=dev)
        g.copy_(grad_ext[:p.n_local])
        if gp.n_rows:
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().pna_halo_grad_pull(self._gtables[self._gcur].data_ptr(), self.n_feat, gp.rows.data_ptr(),
                                                         gp.rowptr.data_ptr(), gp.enc.data_ptr(), gp.shift, gp.n_rows, g.data_ptr(),
                                                         self.n_feat, self.n_feat, torch.cuda.current_stream(dev).cuda_stream))
        self._gcur = (self._gcur + 1) % len(self._gbufs)
        return g

    def return_halo_grad(self, grad_ext: torch.Tensor) -> torch.Tensor:
        """Backward of the exchange: ``stage_halo_grad`` then ``pull_halo_grad`` (one barrier)."""
        self.stage_halo_grad(grad_ext)
        return self.pull_halo_grad(grad_ext)

    def check(self) -> None:
        """Host-side check (synchronises): did every barrier see all peers arrive?"""
        _refuse_capture(self)
        if int(self._status.item()) != 0:
            raise RuntimeError("pna_peer_barrier timed out: a peer rank did not reach the barrier")


def _symmetric_tensor(shape, dtype, dev, rank: int, world: int, group):
    """A tensor of `shape` on every rank, each mapped into every process; (local tensor, per-rank pointers, keepalive)."""
    numel = 1
    for d in shape:
        numel *= int(d)
    rows = _symmetric_rows(1, max(numel, 1), dtype, dev, rank, world, group)
    return rows[0].view(-1)[:numel].view(*shape), rows[1], rows[2]


class PeerAggregator:
    """Gather fused with the exchange: remote rows are read over NVLink inside the aggregation kernel.

    Protocol: every rank writes its rows into ``x_local`` -> ``barrier()`` -> ``aggregate()``.  The barrier orders "all ranks
    have written" before the gathers; NOTHING orders the end of the peers' gathers before this rank's next write into
    ``x_local`` -- a rank that finishes ``aggregate()`` early must not overwrite its rows while slower peers may still be
    reading them.  Either call ``barrier()`` again after ``aggregate()`` before rewriting ``x_local`` (what a multi-layer net
    using ONE buffer has to do), or alternate between two aggregators / buffers per layer as ``PullAggregator`` does
    (``flip()``), where the next layer's barrier separates this layer's reads from the writes two layers later.

    Training (``trainable=True``; opt-in, a forward-only aggregator allocates and communicates nothing more):
    ``pna_aggregate(x, ...)`` is differentiable in ``x`` and ``row_bias``.  Forward: ``x`` is copied into the next slot of a
    ring of ``saved_layers`` symmetric row buffers (allocated once, collectively), a device barrier
    (``pna_peer_barrier``), then the peer forward from that slot's pointer table.  The slot stays readable by the peers until
    their backward has read it.  Backward, per feature slab (``aggregate.deterministic_slab_width`` of the largest rank's
    slot count): ``pna_aggregate_bwd_peer_slots`` stores the gradient of every slot of this rank's CSR into its symmetric
    fp32 per-slot buffer, reading the source rows from the saved slot over NVLink; a barrier; then every owner adds the
    slots that gather its rows into a zeroed ``[n_local, F]`` gradient with ``pna_halo_grad_pull``, in ascending
    (rank, slot) order -- the slot order of the whole graph's CSR (``peer_grad_return_plan``).  Rows nobody gathers get zero.

    Reuse.  A rank rewrites a saved slot or a per-slot buffer only after a barrier that no peer enters before its last read
    of it.  Per-slot buffers alternate (two of them): slab step j+2 rewrites the buffer peers pulled from in step j only
    after this rank has passed the barrier of step j+1, which no peer enters before its pull of step j is done.  A ring
    slot written by call i is rewritten by call i + saved_layers, after this rank has passed the barriers of (a) call
    i + saved_layers - 1 (saved_layers >= 2), which no peer enters before its forward gathers of call i are done, and (b) the
    last slab of call i's backward, which no peer enters before its backward kernels of call i are done -- provided that
    backward ran first.  So the caller's rule: every rank makes the same sequence of calls (forward and backward), and at
    most ``saved_layers`` differentiable calls run between backward passes.  A call beyond that raises, and so does a
    backward whose saved slot has been rewritten since its forward.

    Determinism: the backward has no floating-point atomic anywhere (per-slot stores, then sums in a fixed order), so it
    is bit-reproducible whatever ``torch.use_deterministic_algorithms`` says, and it ignores ``PNA_B200_BWD``.  Parameter
    gradients are this rank's partial sums; summing them across ranks (``all_reduce``) is the caller's job.

    ``_alloc(shape, dtype) -> (local tensor, per-rank pointers, keepalive)`` replaces the symmetric allocation (called for
    ``x_local``, then, trainable only, the ring slots, the barrier flags and the two per-slot buffers) and ``_barrier`` the
    device barrier: tests run W ranks in one process through them."""

    def __init__(self, src_global: torch.Tensor, dst_global: torch.Tensor, bounds: torch.Tensor, rank: int, world: int,
                 n_feat: int, dtype=torch.float32, group=None, trainable: bool = False, saved_layers: int = 2,
                 grad_plan: Optional[GradReturnPlan] = None, _alloc=None, _barrier=None):
        dev = src_global.device
        self.rank, self.world, self.group, self.n_feat, self.dtype = rank, world, group, n_feat, dtype
        lo, hi = int(bounds[rank]), int(bounds[rank + 1])
        self.n_local = hi - lo
        self.shift = peer_shift_for(bounds)
        enc = encode_peer_sources(src_global, bounds, self.shift)
        self.csr = build_csr(enc, dst_global - lo, self.n_local, n_src=world << self.shift)
        rows_max = int((bounds[1:] - bounds[:-1]).max())
        if _alloc is None:
            self.x_local, self.peer_ptrs, self._keep = _symmetric_rows(rows_max, n_feat, dtype, dev, rank, world, group)
            alloc = lambda shape, dt: _symmetric_tensor(shape, dt, dev, rank, world, group)  # noqa: E731
        else:
            self.x_local, self.peer_ptrs, self._keep = _alloc((rows_max, n_feat), dtype)
            alloc = _alloc
        self.x_local = self.x_local[: self.n_local]
        self.ptr_table = torch.tensor(self.peer_ptrs, dtype=torch.int64, device=dev)
        self.trainable, self.grad_plan = trainable, None
        if not trainable:
            return
        if saved_layers < 2:
            raise ValueError("saved_layers must be at least 2 (a slot is rewritten only after the next call's barrier)")
        if grad_plan is None:
            col = self.csr.col[: self.csr.n_edges]
            grad_plan = build_peer_grad_return_plan(col, self.shift, rank, world, group) if world > 1 else \
                peer_grad_return_plan(rank, 1, [col.long() & ((1 << self.shift) - 1)],
                                      [torch.arange(col.numel(), device=dev)], [col.numel()], device=dev)
        if grad_plan.rank != rank or grad_plan.world != world:
            raise ValueError("grad_plan belongs to another rank or world")
        if grad_plan.peer_n_edges is None or grad_plan.peer_n_edges[rank] != self.csr.n_edges:
            raise ValueError("grad_plan is not this graph's peer-plane reverse slot plan (peer_grad_return_plan)")
        self.grad_plan = grad_plan
        self._ring, self._ring_tables, self._ring_gen, self._ring_keep = [], [], [], []
        for _ in range(saved_layers):
            t, ptrs, keep = alloc((rows_max, n_feat), dtype)
            self._ring.append(t)
            self._ring_tables.append(torch.tensor(ptrs, dtype=torch.int64, device=dev))
            self._ring_gen.append(0)
            self._ring_keep.append(keep)
        self._next, self._calls_since_backward = 0, 0
        flags, fptrs, keep = alloc((max(world, 1),), torch.int64)
        flags.zero_()
        self._flags, self._flag_table = flags, torch.tensor(fptrs, dtype=torch.int64, device=dev)
        self._ring_keep.append(keep)
        self._status = torch.zeros(1, dtype=torch.int32, device=dev)
        self._epoch = 0
        # per-slot gradient buffers: the same pitch on every rank (the slab width of the largest rank's slot count)
        self._e_max = max(max(grad_plan.peer_n_edges), 1)
        self._slab = deterministic_slab_width(self._e_max, n_feat, 16 // torch.empty(0, dtype=dtype).element_size())
        self._gbufs, self._gtables, self._gcur = [], [], 0
        for _ in range(2):
            t, ptrs, keep = alloc((self._e_max, self._slab), torch.float32)
            self._gbufs.append(t)
            self._gtables.append(torch.tensor(ptrs, dtype=torch.int64, device=dev))
            self._ring_keep.append(keep)
        self._barrier_hook = _barrier
        self._use_device_barrier = _barrier is None and (world > 1 and _alloc is None)
        if self._use_device_barrier:      # flags are zero everywhere before the first flag store can arrive
            torch.cuda.synchronize(dev)
            dist.barrier(group=group, device_ids=[dev.index])

    def barrier(self) -> None:
        """All ranks have finished writing their x rows (device-side, on the current stream)."""
        _refuse_capture(self)
        h = self._keep.get("handle") if isinstance(self._keep, dict) else None
        if h is not None and hasattr(h, "barrier"):
            h.barrier()
        else:
            dist.barrier(group=self.group, device_ids=[self.x_local.device.index])

    def aggregate(self, aggregators, scalers, avg_deg, out: Optional[torch.Tensor] = None, **kw) -> torch.Tensor:
        _refuse_capture(self)
        return aggregate_forward(self.x_local, self.csr, aggregators, scalers, avg_deg, out=out,
                                 peer=(self.ptr_table, self.shift), **kw)

    # ---- differentiable path (trainable=True) ----
    def _sync(self) -> None:
        """The trainable path's barrier: ``pna_peer_barrier`` on the current stream (or the ``_barrier`` hook)."""
        if self._barrier_hook is not None:
            self._barrier_hook()
            return
        if not self._use_device_barrier:
            return
        self._epoch += 1
        dev = self._flags.device
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().pna_peer_barrier(self._flag_table.data_ptr(), self.rank, self.world, self._epoch, 0,
                                                   self._status.data_ptr(), torch.cuda.current_stream(dev).cuda_stream))

    def check(self) -> None:
        """Host-side check (synchronises): did every barrier of the trainable path see all peers arrive?"""
        _refuse_capture(self)
        if self.trainable and int(self._status.item()) != 0:
            raise RuntimeError("pna_peer_barrier timed out: a peer rank did not reach the barrier")

    def pna_aggregate(self, x: torch.Tensor, aggregators, scalers, avg_deg, *, towers: int = 1,
                      row_bias: Optional[torch.Tensor] = None, self_feat: Optional[torch.Tensor] = None,
                      self_divided: bool = True, zero_isolated: bool = False, relu_var: bool = False,
                      scaler_degree: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Differentiable aggregation of this rank's rows, gathered over NVLink: x is the rank's ``[n_local, F]``
        features, ``row_bias`` / ``self_feat`` are per destination and stay local; returns the rank's ``[n_local, width]``
        output.  Needs ``trainable=True``; the rules on the call sequence are in the class docstring."""
        _refuse_capture(self)
        if not self.trainable:
            raise RuntimeError("PeerAggregator.pna_aggregate needs PeerAggregator(..., trainable=True)")
        if tuple(x.shape) != (self.n_local, self.n_feat) or x.dtype != self.dtype:
            raise ValueError(f"x must be [{self.n_local}, {self.n_feat}] {self.dtype}, got {tuple(x.shape)} {x.dtype}")
        if any(a in _lib.MOMENTS + _lib.WEIGHTED for a in _names(aggregators)):
            raise ValueError("the peer plane has no moment, softmax, softmin or normalised_mean aggregators")
        needs_grad = torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, row_bias, self_feat))
        if needs_grad and self._calls_since_backward >= len(self._ring):
            raise RuntimeError(f"more than saved_layers={len(self._ring)} differentiable calls before a backward: the "
                               "oldest saved features would be overwritten")
        slot = self._next
        self._next = (slot + 1) % len(self._ring)
        self._ring_gen[slot] += 1
        self._ring[slot][: self.n_local].copy_(x)
        self._sync()
        kw = dict(towers=towers, self_divided=self_divided, zero_isolated=zero_isolated, relu_var=relu_var,
                  scaler_degree=scaler_degree)
        if not needs_grad:
            return self._aggregate_saved(slot, aggregators, scalers, avg_deg, row_bias, self_feat, kw)
        self._calls_since_backward += 1
        return _PeerAggregate.apply(x, row_bias, self_feat, self, slot, _names(aggregators), _names(scalers), dict(avg_deg), kw)

    def _aggregate_saved(self, slot: int, aggregators, scalers, avg_deg, row_bias, self_feat, kw) -> torch.Tensor:
        return aggregate_forward(self._ring[slot][: self.n_local], self.csr, aggregators, scalers, avg_deg,
                                 row_bias=row_bias, self_feat=self_feat, peer=(self._ring_tables[slot], self.shift), **kw)

    def _backward_slots(self, grad_out: torch.Tensor, slot: int, aggregators, scalers, avg_deg, *, towers: int = 1,
                       row_bias: Optional[torch.Tensor] = None, has_self: bool = False, relu_var: bool = False,
                       scaler_degree: Optional[torch.Tensor] = None, need_bias_grad: bool = False):
        """The backward of the forward run from ring slot ``slot``: (fp32 gradient of this rank's x, fp32 gradient of
        row_bias or None).  Collective: every rank runs it for the same call, in the same order."""
        n, F, csr = self.n_local, self.n_feat, self.csr
        dev = self._ring[slot].device
        x = self._ring[slot][:n]
        n_aggr, aggr_codes = _lib.pack_codes(aggregators, _lib.ALL_AGGR_CODES, "aggregator")
        n_scal, scal_codes = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
        grad_out = _rows2d(grad_out.to(self.dtype), "grad_out")
        if row_bias is not None:
            row_bias = _rows2d(row_bias.to(self.dtype), "row_bias")
        gb = torch.zeros((n, F), dtype=torch.float32, device=dev) if need_bias_grad else None
        d = _lib.AggStruct(
            gathered=x.data_ptr(), ld_gathered=F, rowptr=csr.rowptr.data_ptr(), col=csr.col.data_ptr() if csr.n_edges else None,
            row_bias=None if row_bias is None else row_bias.data_ptr(),
            ld_row_bias=0 if row_bias is None else (row_bias.stride(0) if n > 1 else F),
            self_feat=1 if has_self else None,     # only its presence matters here: it shifts the grad_out columns
            n_rows=n, n_feat=F, n_towers=towers, dtype=_DTYPES[self.dtype],
            n_aggr=n_aggr, aggr_codes=aggr_codes, n_scalers=n_scal, scaler_codes=scal_codes,
            avg_log=float(avg_deg["log"]), avg_lin=float(avg_deg.get("lin", 1.0)),
            flags=_lib.FLAG_RELU_VAR if relu_var else 0, split_threshold=csr.split_threshold, chunk_edges=csr.chunk_edges,
            hub_info=csr.hub_info.data_ptr() if csr.n_hubs else None,
            chunk_items=csr.chunk_items.data_ptr() if csr.n_hubs else None, n_hubs=csr.n_hubs, n_chunks=csr.n_chunks,
            peer_gathered=self._ring_tables[slot].data_ptr(), peer_shift=self.shift)
        if scaler_degree is not None:
            d.scaler_degree = scaler_degree.data_ptr()
        scratch = None
        if csr.n_hubs:
            scratch = torch.empty(((csr.n_chunks + csr.n_hubs) * 6, F), dtype=torch.float32, device=dev)
            d.hub_partials = scratch.data_ptr()
        ld_go = grad_out.stride(0) if n > 1 else grad_out.size(1)
        gp, L = self.grad_plan, _lib.lib()
        g = torch.zeros((n, F), dtype=torch.float32, device=dev)
        for f0 in range(0, F, self._slab):
            fc = min(self._slab, F - f0)
            gs = self._gbufs[self._gcur].view(-1)[: self._e_max * fc].view(self._e_max, fc)
            stream = torch.cuda.current_stream(dev).cuda_stream
            if csr.n_edges:
                with torch.cuda.device(dev):
                    _lib.check(L.pna_aggregate_bwd_peer_slots(C.byref(d), grad_out.data_ptr(), ld_go, f0, fc, gs.data_ptr(), fc,
                                                              None if gb is None else gb.data_ptr(), F, stream))
            self._sync()          # every rank's per-slot gradients of this slab are stored
            if gp.n_rows:
                with torch.cuda.device(dev):
                    _lib.check(L.pna_halo_grad_pull(self._gtables[self._gcur].data_ptr(), fc, gp.rows.data_ptr(),
                                                    gp.rowptr.data_ptr(), gp.enc.data_ptr(), gp.shift, gp.n_rows,
                                                    g[:, f0:].data_ptr(), F, fc, stream))
            self._gcur = (self._gcur + 1) % len(self._gbufs)
        return g, gb


class _PeerAggregate(torch.autograd.Function):
    """The peer plane's differentiable aggregation (``PeerAggregator.pna_aggregate``): x lives in a ring slot of the
    aggregator, which the backward reads through the peers' pointer table."""

    @staticmethod
    def forward(ctx, x, row_bias, self_feat, agg, slot, aggregators, scalers, avg_deg, kw):
        out = agg._aggregate_saved(slot, aggregators, scalers, avg_deg, row_bias, self_feat, kw)
        ctx.save_for_backward(row_bias, self_feat)
        ctx.meta = (agg, slot, agg._ring_gen[slot], aggregators, scalers, avg_deg, kw, x.dtype)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        row_bias, self_feat = ctx.saved_tensors
        agg, slot, gen, aggregators, scalers, avg_deg, kw, x_dtype = ctx.meta
        if agg._ring_gen[slot] != gen:
            raise RuntimeError("the saved features of this peer-plane call were overwritten by a later call before its "
                               f"backward: at most saved_layers={len(agg._ring)} differentiable calls between backward passes")
        agg._calls_since_backward = 0
        towers = kw["towers"]
        g, gb = agg._backward_slots(grad_out, slot, aggregators, scalers, avg_deg, towers=towers, row_bias=row_bias,
                                   has_self=self_feat is not None, relu_var=kw["relu_var"],
                                   scaler_degree=kw["scaler_degree"], need_bias_grad=ctx.needs_input_grad[1])
        gs = None
        if self_feat is not None and ctx.needs_input_grad[2]:
            # the self block of every tower is a plain copy: its gradient is the matching slice of grad_out
            N, F = agg.n_local, agg.n_feat
            Ft = F // towers
            blk = grad_out.reshape(N, towers, -1)[:, :, :Ft]
            gs = (blk.reshape(N, F) if kw["self_divided"] else blk.sum(1)).to(self_feat.dtype)
        return (g.to(x_dtype) if ctx.needs_input_grad[0] else None, None if gb is None else gb.to(row_bias.dtype), gs,
                None, None, None, None, None, None)


def _symmetric_rows(rows: int, n_feat: int, dtype, dev, rank: int, world: int, group):
    """A [rows, n_feat] buffer on every rank, each mapped into every process; returns (local tensor, pointers, keepalive)."""
    try:
        import torch.distributed._symmetric_memory as symm
        t = symm.empty((rows, n_feat), dtype=dtype, device=dev)
        h = symm.rendezvous(t, group=group if group is not None else dist.group.WORLD)
        ptrs = [int(p) for p in h.buffer_ptrs]
        return t, ptrs, {"handle": h, "tensor": t, "how": "torch symmetric memory"}
    except Exception as exc:  # CUDA IPC fallback: share the caching-allocator block, open it on every peer
        t = torch.empty((rows, n_feat), dtype=dtype, device=dev)
        meta = t.untyped_storage()._share_cuda_()
        metas = [None] * world
        dist.all_gather_object(metas, meta, group=group)
        opened, ptrs = [], []
        for r in range(world):
            if r == rank:
                ptrs.append(t.data_ptr())
                continue
            st = torch.UntypedStorage._new_shared_cuda(*metas[r])
            peer = torch.empty(0, dtype=dtype, device=st.device).set_(st, 0, (rows, n_feat), (n_feat, 1))
            opened.append((st, peer))
            ptrs.append(peer.data_ptr())
        return t, ptrs, {"opened": opened, "tensor": t, "how": f"CUDA IPC (symmetric memory unavailable: {exc})"}


# ---- synthetic destination-partitioned workload (tools/dist_check.py; the bench lines come from bench_multi.py) ------
def rank_graph(rank: int, world: int, n_local: int, e_local: int, n_feat: int, p_remote: float, seed: int = 0,
               skew: float = 3.0, dtype=torch.float32):
    """In-edges of rank's rows in a graph of world * n_local nodes: destinations skewed like synth.arxiv_like inside
    the rank's range; a source is drawn from the whole graph with probability p_remote, else from the rank's range."""
    g = torch.Generator().manual_seed(seed * 1000 + rank)
    lo = rank * n_local
    perm = torch.randperm(n_local, generator=g)
    u = torch.rand(e_local, generator=g, dtype=torch.float64)
    dst = lo + perm[(n_local * u.pow(skew)).long().clamp_(max=n_local - 1)]
    local_src = lo + torch.randint(0, n_local, (e_local,), generator=g)
    any_src = torch.randint(0, world * n_local, (e_local,), generator=g)
    src = torch.where(torch.rand(e_local, generator=g) < p_remote, any_src, local_src)
    x = torch.randn(n_local, n_feat, generator=g).to(dtype)
    return src, dst, x
