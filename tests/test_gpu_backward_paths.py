"""The aggregation backward's data-selected paths against the exact fp32 restatement (backward_paths_ref.py).

pna_aggregate_bwd picks its kernel instance from the data: row width and alignment (bwd_entry's vec_ok, then
launch_bwd_typed's lane group G and gridDim.y), rows at or above the split threshold (the k_bwd_hub_* chain), the per-slot /
atomic / coefficient entry point, the feature slab, and the alignment of the output rows (gs_vec, vec_atomics, coef_vec).
Each case names the instance it is meant to reach, k_bwd_rows<T, VEC, G, SLOTS>, and asserts a probe that shows the path
ran.  Outputs the kernel writes start as NaN: grad_slots, grad_row_bias and, in the coefficient mode, columns [0, F) and
[c1, c1 + F) of the coefficient rows of rows with in-edges.  Rows without in-edges get no coefficient row (the transposed
sum never reads it), so theirs is not required.  Per-slot values, coefficient rows, closed-form and per-slot-instance
row-bias gradients, the transposed sums and the deterministic grad_gathered must match bit for bit.  Sums the atomics form
must lie within the rigorous order-free bound of their float64 value.  The degree-scaler factors are the library's own
(pna_row_scales), never a host logarithm.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import backward_paths_ref as B
import forward_paths_ref as FR

pytestmark = pytest.mark.gpu

A6 = ["sum", "mean", "min", "max", "var", "std"]
S3 = ["identity", "amplification", "attenuation"]
S5 = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]


@pytest.fixture(scope="module")
def P():
    import pna_b200
    return pna_b200


def dev():
    return torch.device("cuda:0")


def np32(t):
    return None if t is None else t.float().cpu().numpy()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def assert_bits(got, want, what=""):
    g, w = bits(got), bits(want)
    bad = g != w
    assert not bad.any(), f"{what}: {int(bad.sum())} elements differ, first {np.argwhere(bad)[:4].tolist()}"


# ---- graphs ---------------------------------------------------------------------------------------------------------------
_GRAPHS = {}


def gpu_csr(P, key, make, split=None, chunk=None):
    if key not in _GRAPHS:
        src, dst, n = make()
        csr = P.build_csr(torch.from_numpy(src).to(dev()), torch.from_numpy(dst).to(dev()), n, split, chunk)
        host = (csr.rowptr.cpu().numpy().astype(np.int64), csr.col.cpu().numpy().astype(np.int64),
                csr.hub_info.cpu().numpy().astype(np.int64).reshape(-1, 4), csr.chunk_items.cpu().numpy().astype(np.int64).reshape(-1, 2))
        _GRAPHS[key] = (csr, host)
    return _GRAPHS[key]


def host_of(csr):
    return (csr.rowptr.cpu().numpy().astype(np.int64), csr.col.cpu().numpy().astype(np.int64),
            csr.hub_info.cpu().numpy().astype(np.int64).reshape(-1, 4), csr.chunk_items.cpu().numpy().astype(np.int64).reshape(-1, 2))


def mixed(split=256, chunk=128, n=700, e=5000, seed=1):
    """random in-edges into rows 10 .. n-21, rows 0..3 of degree split-1, split, k*chunk, k*chunk+1 (k the smallest with
    k*chunk > split), row 4 several chunks more; the last 20 rows isolated"""
    def make():
        rng = np.random.default_rng(seed)
        k = split // chunk + 1
        fixed = {0: split - 1, 1: split, 2: k * chunk, 3: k * chunk + 1, 4: split + 3 * chunk + 5}
        dst = np.concatenate([rng.integers(10, n - 20, e)] + [np.full(d, r) for r, d in fixed.items()])
        src = rng.integers(0, n, dst.size)
        p = rng.permutation(dst.size)
        return src[p], dst[p], n
    return make


def zipf(n=3000, e=30000, seed=2):
    """Zipf-distributed sources (the hottest ones are split rows of the transposed CSRs), uniform destinations plus two split
    rows; the last 50 rows isolated"""
    def make():
        rng = np.random.default_rng(seed)
        src = (rng.zipf(1.4, e + 900) - 1) % n
        dst = np.concatenate([rng.integers(0, n - 52, e), np.full(300, n - 52), np.full(600, n - 51)])
        return src, dst, n
    return make


def identical(n=400, seed=3):
    """rows 0..39 gather one source 2..40 times (identical messages: var <= 0), row 40 gathers one source 300 times (a split
    row of identical messages), random rows 50.. beside them"""
    def make():
        rng = np.random.default_rng(seed)
        dst = [np.full(2 + r, r) for r in range(40)] + [np.full(300, 40), rng.integers(50, n, 3000)]
        src = [np.full(2 + r, 100 + r) for r in range(40)] + [np.full(300, 7), rng.integers(0, n, 3000)]
        return np.concatenate(src), np.concatenate(dst), n
    return make


def avg_of(csr):
    deg = csr.in_degree.long().cpu()
    hist = torch.bincount(deg).double()
    b = torch.arange(hist.numel(), dtype=torch.float64)
    return {"log": float(((b + 1).log() * hist).sum() / hist.sum()), "lin": float((b * hist).sum() / hist.sum())}


def rand(shape, dtype, seed, layout="contig", ints=None):
    """[n, f] on the GPU; "pitch+2" = view of an [n, f+2] buffer (odd pitch), "offset1" = columns 1..f of [n, f+4]
    (misaligned base), ("wide", k) = the first f columns of [n, f+k]"""
    n, f = shape
    g = torch.Generator().manual_seed(seed)
    extra, lo = {"contig": (0, 0), "pitch+2": (2, 0), "offset1": (4, 1)}.get(layout, (layout[1] if isinstance(layout, tuple) else 0, 0))
    t = torch.randint(-ints, ints + 1, (n, f + extra), generator=g).float() if ints else torch.randn(n, f + extra, generator=g)
    return t.to(dtype).to(dev())[:, lo:lo + f]


def scales_of(P, csr, scalers, avg, sdeg=None):
    """[N, S] fp32 factors the kernel multiplies by: pna_row_scales of the in-degree, or of scaler_degree (a rowptr built from it)"""
    if sdeg is None:
        return P.aggregate.row_scales(csr, scalers, avg).cpu().numpy()
    from pna_b200 import _lib
    rp = torch.zeros(csr.n_nodes + 1, dtype=torch.int32, device=dev())
    rp[1:] = torch.cumsum(sdeg.long(), 0).int()
    ns, codes = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
    out = torch.empty((csr.n_nodes, ns), dtype=torch.float32, device=dev())
    _lib.check(_lib.lib().pna_row_scales(rp.data_ptr(), csr.n_nodes, ns, codes, float(avg["log"]), float(avg["lin"]), out.data_ptr(),
                                         torch.cuda.current_stream().cuda_stream))
    return out.cpu().numpy()


class Call:
    """One direct call into the backward ABI: descriptor, grad_out, scratch, and the exact reference of the same call."""

    def __init__(self, P, csr, host, x, go, aggrs, scalers, avg, *, towers=1, bias=None, has_self=False, relu_var=False,
                 sdeg=None, messages=None, reference_of=None):
        from pna_b200 import _lib
        self.L, self.lib = _lib.lib(), _lib
        self.csr, self.host, self.x, self.go, self.bias = csr, host, x, go, bias
        self.n, self.f = csr.n_nodes, x.size(1)
        self.aggrs, self.scalers, self.towers, self.has_self = aggrs, scalers, towers, has_self
        self.relu_var, self.sdeg = relu_var, sdeg
        self.scratch = torch.full(((csr.n_chunks + csr.n_hubs) * 6 + 1, self.f), float("nan"), device=dev())
        g = messages if messages is not None else x
        na, ac = _lib.pack_codes(aggrs, _lib.AGGR_CODES, "aggregator")
        ns, sc = _lib.pack_codes(scalers, _lib.SCALER_CODES, "scaler")
        self.d = _lib.AggStruct(
            gathered=g.data_ptr(), ld_gathered=g.stride(0), rowptr=csr.rowptr.data_ptr(),
            col=None if messages is not None else csr.col.data_ptr(), row_bias=None if bias is None else bias.data_ptr(),
            ld_row_bias=0 if bias is None else bias.stride(0), self_feat=1 if has_self else None, n_rows=self.n, n_feat=self.f,
            n_towers=towers, dtype=_lib.PNA_F32 if x.dtype == torch.float32 else _lib.PNA_BF16, n_aggr=na, aggr_codes=ac,
            n_scalers=ns, scaler_codes=sc, avg_log=float(avg["log"]), avg_lin=float(avg["lin"]),
            flags=_lib.FLAG_RELU_VAR if relu_var else 0, split_threshold=csr.split_threshold, chunk_edges=csr.chunk_edges,
            hub_info=csr.hub_info.data_ptr() if csr.n_hubs else None, chunk_items=csr.chunk_items.data_ptr() if csr.n_hubs else None,
            n_hubs=csr.n_hubs, n_chunks=csr.n_chunks, hub_partials=self.scratch.data_ptr())
        if sdeg is not None:
            self.d.scaler_degree = sdeg.data_ptr()
        self.gathered = g
        esz = x.element_size()
        rows = [(g.data_ptr(), g.stride(0)), (go.data_ptr(), go.stride(0))] + ([] if bias is None else [(bias.data_ptr(), bias.stride(0))])
        self.vec_ok = B.bwd_vec_ok(self.f // towers, esz, rows)
        self.deg = np.diff(host[0])
        if reference_of is not None:      # the same inputs, another entry point or layout: the same reference
            for k in ("st", "scales", "c", "gm", "gb", "shares"):
                setattr(self, k, getattr(reference_of, k))
            return
        rowptr, col, info, _ = host
        xn, bn = np32(x), np32(bias)
        self.st = B.row_stats_bwd(xn, rowptr, col, info, csr.chunk_edges, bn)
        self.scales = scales_of(P, csr, scalers, avg, sdeg)
        self.c = B.coefficients(self.st, self.deg, np32(go), self.scales, aggrs, towers=towers, has_self=has_self, relu_var=relu_var)
        self.gm, self.gb, self.shares = B.slot_grads(self.c, self.st, xn, rowptr, col, info, csr.chunk_edges, bn)

    def stream(self):
        return torch.cuda.current_stream().cuda_stream

    def instance(self, width=None):
        return B.bwd_instance(self.f if width is None else width, self.x.element_size(), self.vec_ok)

    def slots(self, f0=0, fc=None, ld_extra=0):
        fc = self.f - f0 if fc is None else fc
        E = self.csr.n_edges
        ld = fc + ld_extra
        gs = torch.full((max(E, 1), ld), float("nan"), device=dev())
        gb = torch.full((self.n, self.f), float("nan"), device=dev())
        self.lib.check(self.L.pna_aggregate_bwd_slots(C.byref(self.d), self.go.data_ptr(), self.go.stride(0), f0, fc, gs.data_ptr(), ld,
                                                      gb.data_ptr(), self.f, self.stream()))
        return gs[:E, :fc].cpu().numpy(), gb.cpu().numpy()

    def atomic(self, ld_extra=0):
        n_src = self.gathered.size(0)
        gg = torch.zeros((n_src, self.f + ld_extra), device=dev())
        gb = torch.full((self.n, self.f), float("nan"), device=dev())
        self.lib.check(self.L.pna_aggregate_bwd(C.byref(self.d), self.go.data_ptr(), self.go.stride(0), gg.data_ptr(), gg.stride(0),
                                                gb.data_ptr(), self.f, self.stream()))
        return gg[:, :self.f].cpu().numpy(), gb.cpu().numpy()

    def split_rows(self):
        return self.host[2][:, 0]

    def light_rows(self):
        m = np.ones(self.n, bool)
        m[self.split_rows()] = False
        return m

    def check_bias_atomic(self, gb):
        """grad_row_bias of the atomic instance: light rows in slot order (exact), split rows' chunk shares in any order"""
        lr = self.light_rows()
        assert_bits(gb[lr], self.gb[lr], "grad_row_bias, light rows")
        if self.csr.n_hubs:
            crow, _, _ = B.chunk_bounds(self.host[0], self.host[2], self.csr.chunk_edges)
            s, bound = B.order_free_sum(self.n, crow, self.shares)
            r = self.split_rows()
            assert B.within_order_free(gb[r], s[r], bound[r]).all()


def make_call(P, graph, f, dtype, seed, aggrs=A6, scalers=S3, layout="contig", go_extra=0, bias=True, towers=1, has_self=False,
              ints=None, **kw):
    csr, host = graph
    n = csr.n_nodes
    x = rand((n, f), dtype, seed, layout, ints)
    b = rand((n, f), dtype, seed + 1, ints=ints) if bias else None
    width = towers * (int(has_self) + len(aggrs) * len(scalers)) * (f // towers)
    go = rand((n, width), dtype, seed + 2, ("wide", go_extra) if go_extra else "contig", ints)
    return Call(P, csr, host, x, go, aggrs, scalers, avg_of(csr), towers=towers, bias=b, has_self=has_self, **kw)


def check_slots_and_stores(P, call):
    """pna_aggregate_bwd_slots and pna_aggregate_bwd with col == NULL (messages in CSR order: grad_gathered[slot] is STORED)
    give the restatement's per-slot values; grad_row_bias as each instance forms it"""
    gs, gb = call.slots()
    assert_bits(gs, call.gm, "grad_slots")
    assert_bits(gb, call.gb, "grad_row_bias (per-slot instance)")
    xm = call.x[call.csr.col.long()].contiguous()
    c2 = Call(P, call.csr, call.host, call.x, call.go, call.aggrs, call.scalers, avg_of(call.csr), towers=call.towers,
              bias=call.bias, has_self=call.has_self, relu_var=call.relu_var, sdeg=call.sdeg, messages=xm, reference_of=call)
    gg, gb2 = c2.atomic()
    assert_bits(gg, call.gm, "grad_gathered stores (col == NULL)")
    call.check_bias_atomic(gb2)


# ---- 1. lane groups and widths --------------------------------------------------------------------------------------------
WIDTHS = [
    # F, dtype, bias, (VEC, G, gridDim.y)      instance
    (4, torch.float32, True, (4, 1, 1)),        # k_bwd_rows<float,4,1,SLOTS> + k_bwd_hub_{stats,coef,scatter,bias}<float,4,1>
    (8, torch.float32, False, (4, 2, 1)),       # k_bwd_rows<float,4,2,SLOTS> + hub chain
    (16, torch.float32, True, (4, 4, 1)),       # k_bwd_rows<float,4,4,SLOTS>
    (32, torch.float32, False, (4, 8, 1)),      # k_bwd_rows<float,4,8,SLOTS>
    (64, torch.float32, True, (4, 16, 1)),      # k_bwd_rows<float,4,16,SLOTS>
    (128, torch.float32, False, (4, 32, 1)),    # k_bwd_rows<float,4,32,SLOTS>
    (256, torch.float32, True, (4, 32, 2)),     # k_bwd_rows<float,4,32,SLOTS>, gridDim.y = 2
    (1024, torch.float32, False, (4, 32, 8)),   # k_bwd_rows<float,4,32,SLOTS>, gridDim.y = 8
    (8, torch.bfloat16, True, (8, 1, 1)),       # k_bwd_rows<bf16,8,1,SLOTS>
    (64, torch.bfloat16, False, (8, 8, 1)),     # k_bwd_rows<bf16,8,8,SLOTS>
    (256, torch.bfloat16, True, (8, 32, 1)),    # k_bwd_rows<bf16,8,32,SLOTS>
    (512, torch.bfloat16, False, (8, 32, 2)),   # k_bwd_rows<bf16,8,32,SLOTS>, gridDim.y = 2
]


@pytest.mark.parametrize("f,dtype,bias,inst", WIDTHS)
def test_lane_groups_and_widths(P, f, dtype, bias, inst):
    call = make_call(P, gpu_csr(P, "mixed", mixed()), f, dtype, seed=f, bias=bias)
    assert call.csr.n_hubs >= 4 and call.vec_ok and call.instance() == inst
    check_slots_and_stores(P, call)


# ---- 2. scalar fallbacks (VEC = 1) ----------------------------------------------------------------------------------------
SCALAR = [
    # F, dtype, towers, layout, extra grad_out columns          instance
    (75, torch.float32, 3, "pitch+2", 0),     # k_bwd_rows<float,1,32,SLOTS>, gridDim.y = 3, odd pitch, 3 towers + self block
    (75, torch.float32, 3, "offset1", 0),     # k_bwd_rows<float,1,32,SLOTS>, misaligned base
    (75, torch.float32, 3, "contig", 7),      # k_bwd_rows<float,1,32,SLOTS>, ld_grad_out = T*Wt + 7
    (96, torch.float32, 3, "contig", 2),      # k_bwd_rows<float,1,32,SLOTS>: Ft = 32, scalar only because of ld_grad_out
    (48, torch.bfloat16, 3, "offset1", 0),    # k_bwd_rows<bf16,1,32,SLOTS>, gridDim.y = 2, misaligned base
]


@pytest.mark.parametrize("f,dtype,towers,layout,go_extra", SCALAR)
def test_scalar_fallbacks(P, f, dtype, towers, layout, go_extra):
    call = make_call(P, gpu_csr(P, "mixed", mixed()), f, dtype, seed=f + go_extra, layout=layout, go_extra=go_extra,
                     towers=towers, has_self=True)
    assert not call.vec_ok and call.instance()[0] == 1 and call.csr.n_hubs > 0
    if go_extra == 2:   # the probe: only the grad_out pitch turns the vector path off
        assert (f // towers) % 4 == 0 and call.go.stride(0) % 4 != 0
    check_slots_and_stores(P, call)


# ---- 3. split rows --------------------------------------------------------------------------------------------------------
def _ties_straddle_chunks(call):
    """the probe: some split row's minimum (maximum) occurs in two different chunks"""
    rowptr, col, info, _ = call.host
    x, b = np32(call.x), np32(call.bias)
    ch = call.csr.chunk_edges
    for r, _, _, d in info:
        m = x[col[rowptr[r]:rowptr[r + 1]]] + (b[r] if b is not None else 0)
        chunk = np.arange(d) // ch
        for ext in (m.min(0), m.max(0)):
            for f in range(m.shape[1]):
                if np.unique(chunk[m[:, f] == ext[f]]).size > 1:
                    return True
    return False


SPLIT_CASES = [
    # (split, chunk), dtype, ties      instance
    ((256, 128), torch.float32, False),  # k_bwd_rows<float,4,8> + k_bwd_hub_stats/coef/scatter<float,4,8> + k_bwd_hub_bias<4,8>
    ((256, 128), torch.bfloat16, False),  # k_bwd_rows<bf16,8,8> + hub chain
    ((16, 4), torch.float32, False),     # small chunks: many chunks per split row
    ((16, 4), torch.bfloat16, False),
    ((256, 128), torch.float32, True),   # integer data: ties within and across chunks
    ((256, 128), torch.bfloat16, True),  # bf16 min / max routing
    ((16, 4), torch.float32, True),
    ((16, 4), torch.bfloat16, True),
]


@pytest.mark.parametrize("sc,dtype,ties", SPLIT_CASES)
def test_split_rows(P, sc, dtype, ties):
    split, chunk = sc
    graph = gpu_csr(P, f"mixed{split}", mixed(split, chunk, n=400, e=3000, seed=split), split, chunk)
    f = 32 if dtype == torch.float32 else 64
    call = make_call(P, graph, f, dtype, seed=split + f, aggrs=A6, scalers=S3, ints=2 if ties else None)
    deg = call.deg
    assert call.csr.n_hubs > 0 and deg[0] == split - 1 and 0 not in call.split_rows() and 1 in call.split_rows()
    assert {2, 3} <= set(call.split_rows().tolist()) and deg[2] % chunk == 0 and deg[3] % chunk == 1
    if ties:
        assert _ties_straddle_chunks(call)
    else:   # the probe of k_bwd_hub_bias's order: adding the chunk shares in reverse order changes some bits
        rev = np.zeros_like(call.gb)
        c = 0
        for r, _, nch, _ in call.host[2]:
            acc = np.zeros(f, np.float32)
            for j in range(c + nch - 1, c - 1, -1):
                acc = acc + call.shares[j]
            rev[r] = acc
            c += nch
        r = call.split_rows()
        assert (bits(rev[r]) != bits(call.gb[r])).any()
    gs, gb = call.slots()
    assert_bits(gs, call.gm, "grad_slots")
    assert_bits(gb, call.gb, "grad_row_bias (k_bwd_hub_bias order)")
    # the atomic instance through col: grad_gathered and the split rows' grad_row_bias are order-free sums
    gg, gb2 = call.atomic()
    s, bound = B.order_free_sum(call.n, call.host[1], call.gm)
    assert B.within_order_free(gg, s, bound).all()
    call.check_bias_atomic(gb2)


# ---- 4. feature slabs -----------------------------------------------------------------------------------------------------
SLABS = [
    # F, dtype, f_begin, f_count, extra grad_slots columns     instance
    (256, torch.float32, 128, 64, 0),    # k_bwd_rows<float,4,16,true>, slab [128, 192)
    (256, torch.float32, 192, 64, 3),    # the last of 96-wide slabs; ld_grad_slots = 67: gs_vec off
    (256, torch.float32, 0, 96, 1),      # k_bwd_rows<float,4,32,true>, ld_grad_slots = 97
    (203, torch.float32, 200, 3, 0),     # k_bwd_rows<float,1,4,true>: ragged last slab of a scalar row
    (512, torch.bfloat16, 256, 128, 2),  # k_bwd_rows<bf16,8,16,true>, gs_vec off
    (512, torch.bfloat16, 384, 128, 0),  # k_bwd_rows<bf16,8,16,true>, last slab
]


@pytest.mark.parametrize("f,dtype,f0,fc,ld_extra", SLABS)
def test_feature_slabs(P, f, dtype, f0, fc, ld_extra):
    call = make_call(P, gpu_csr(P, "mixed", mixed()), f, dtype, seed=f + f0, aggrs=["mean", "max", "std"], scalers=S3)
    assert call.csr.n_hubs > 0
    vec = call.instance(fc)[0]
    assert vec == (1 if f % 4 else 16 // call.x.element_size())
    gs, gb = call.slots(f0, fc, ld_extra)
    assert_bits(gs, call.gm[:, f0:f0 + fc], "grad_slots slab")
    assert_bits(gb[:, f0:f0 + fc], call.gb[:, f0:f0 + fc], "grad_row_bias slab")
    outside = np.ones(f, bool)
    outside[f0:f0 + fc] = False
    assert np.isnan(gb[:, outside]).all()        # grad_row_bias is written in the slab's columns only


# ---- 5. flags and inputs --------------------------------------------------------------------------------------------------
FLAG_CASES = [
    # graph, F, dtype, aggregators, scalers, options           instance
    ("identical", 32, torch.float32, ["var", "std", "mean"], S3, {"relu_var": True}),   # k_bwd_rows<float,4,8,*>, PNA_FLAG_RELU_VAR
    ("identical", 64, torch.bfloat16, ["var", "std", "mean"], S3, {"relu_var": True}),  # k_bwd_rows<bf16,8,8,*>
    ("identical", 32, torch.float32, ["var", "std", "mean"], S3, {}),                   # without the flag: var <= 0 still has a slope
    ("mixed", 64, torch.float32, A6, S5, {"sdeg": True}),     # scaler_degree != in-degree, all five scalers
    ("mixed", 64, torch.bfloat16, A6, S5, {"sdeg": True}),
    ("mixed", 32, torch.float32, A6, S5, {}),                 # all five scalers of the in-degree
    ("mixed", 32, torch.float32, ["mean", "_skip", "min", "std", "_skip", "var"], S3, {}),   # PNA_AGGR_SKIP entries
]


@pytest.mark.parametrize("gname,f,dtype,aggrs,scalers,opt", FLAG_CASES)
def test_flags_and_inputs(P, gname, f, dtype, aggrs, scalers, opt):
    graph = gpu_csr(P, gname, identical() if gname == "identical" else mixed())
    csr = graph[0]
    kw = {}
    if opt.get("relu_var"):
        kw["relu_var"] = True
    if opt.get("sdeg"):
        g = torch.Generator().manual_seed(f)
        sdeg = torch.randint(0, 40, (csr.n_nodes,), generator=g, dtype=torch.int32)
        sdeg[::7] = 0
        kw["sdeg"] = sdeg.to(dev())
    call = make_call(P, graph, f, dtype, seed=f + 7, aggrs=aggrs, scalers=scalers, **kw)
    assert csr.n_hubs > 0
    if gname == "identical":   # the probe: rows whose variance is not positive, and the flag changes their coefficients
        mean = call.st[0] / np.maximum(call.deg, 1)[:, None].astype(np.float32)
        var = call.st[1] / np.maximum(call.deg, 1)[:, None].astype(np.float32) - mean * mean
        assert (var[:41] <= 0).any() and 40 in call.split_rows()
        other = B.coefficients(call.st, call.deg, np32(call.go), call.scales, aggrs, relu_var=not opt.get("relu_var"))
        assert (bits(other[1]) != bits(call.c[1])).any()
    if opt.get("sdeg"):        # the probe: the scalers see another degree, and that changes the coefficients
        assert (kw["sdeg"].cpu().numpy() != call.deg).mean() > 0.5
        other = B.coefficients(call.st, call.deg, np32(call.go), scales_of(P, csr, scalers, avg_of(csr)), aggrs)
        assert (bits(other[0]) != bits(call.c[0])).any()
    check_slots_and_stores(P, call)


# ---- 6. coefficient mode through the Python path (PNA_B200_BWD=coef) -------------------------------------------------------
def _spy(P, monkeypatch):
    seen = []
    real = P.aggregate.aggregate_forward

    def spy(gathered, *a, **k):
        out = real(gathered, *a, **k)
        seen.append((gathered.clone(), out.clone()))
        return out
    monkeypatch.setattr(P.aggregate, "aggregate_forward", spy)
    return seen


def _check_grad_gathered_coef(call, gg, s0, s1):
    """grad_gathered = fl(routed + fl(s0 + fl(x*s1))): exact where a (source, feature) receives at most one routed min / max
    term, within the order-free bound elsewhere.  Returns how many elements had 1 and > 1 routed terms."""
    r, f, v = B.routed_terms(call.c, call.st, call.deg, call.host[1])
    R = np.zeros(gg.shape, np.float32)
    np.add.at(R, (r, f), v)          # fp32 per element: exact where at most one term lands
    want = B.combine(R, s0, s1, np32(call.x))
    s, bound, k = B.order_free_sum_elements(gg.shape, r, f, v, base=s0 + np32(call.x) * s1)
    one = k <= 2
    assert_bits(gg[one], want[one], "grad_gathered, at most one routed term")
    assert B.within_order_free(gg[~one], s[~one], bound[~one]).all()
    return int((k == 2).sum()), int((k > 2).sum())


COEF_CASES = [
    # F, dtype, bias, aggregators          instance
    (64, torch.float32, True, A6),         # k_bwd_rows<float,4,16,false> + k_bwd_hub_stats/coef<float,4,16,false> (coef mode)
    (64, torch.bfloat16, True, A6),        # k_bwd_rows<bf16,8,8,false> + hub chain, bf16 routing
    (75, torch.float32, False, A6),        # k_bwd_rows<float,1,32,false>, Fp = 76
    (128, torch.float32, True, ["mean", "var", "std", "sum"]),   # no min / max: grad_gathered exact everywhere
]


@pytest.mark.parametrize("f,dtype,bias,aggrs", COEF_CASES)
def test_coefficient_mode_python_path(P, monkeypatch, f, dtype, bias, aggrs):
    graph = gpu_csr(P, "zipf", zipf())
    csr = graph[0]
    call = make_call(P, graph, f, dtype, seed=f + 11, aggrs=aggrs, scalers=S3, bias=bias)
    tcsr = csr.transposed(csr.n_nodes)
    assert csr.n_hubs > 0 and tcsr.n_hubs > 0 and not csr.sources_unique
    monkeypatch.setenv("PNA_B200_BWD", "coef")
    seen = _spy(P, monkeypatch)
    gg, gb = P.aggregate.aggregate_backward(call.go, call.x, csr, aggrs, S3, avg_of(csr), row_bias=call.bias, need_bias_grad=bias)
    assert len(seen) == 1
    coef, sums = (t.cpu().numpy() for t in seen[0])
    Fp = (f + 3) // 4 * 4
    has_in = call.deg > 0
    assert (~has_in).any()
    c0p, c1, gb_closed = B.coef_rows(call.c, call.st, call.deg, np32(call.bias))
    assert_bits(coef[has_in, :f], c0p[has_in], "c0'")
    assert_bits(coef[has_in, Fp:Fp + f], c1[has_in], "c1")
    if bias:
        gbn = gb.cpu().numpy()
        assert_bits(gbn[has_in], gb_closed[has_in], "closed-form grad_row_bias")
        assert (gbn[~has_in] == 0).all()
    rows = np.zeros((csr.n_nodes, 2 * Fp), np.float32)
    rows[:, :f], rows[:, Fp:Fp + f] = c0p, c1
    want_sums, merge = B.transposed_sums(rows, host_of(tcsr), tcsr.chunk_edges, 2 * Fp, True)
    assert_bits(sums[:, :f], want_sums[:, :f], f"S0 ({merge})")
    assert_bits(sums[:, Fp:Fp + f], want_sums[:, Fp:Fp + f], f"S1 ({merge})")
    one, many = _check_grad_gathered_coef(call, gg.cpu().numpy(), want_sums[:, :f], want_sums[:, Fp:Fp + f])
    if "min" in aggrs:   # the probe: both kinds of element occur
        assert one > 0 and many > 0
    else:
        assert one == 0 and many == 0


# ---- 7. coefficient mode, direct ABI call: scalar stores and scalar atomics; k_bwd_combine -----------------------------------
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_coefficient_mode_direct_call(P, dtype):
    # k_bwd_rows<T,VEC,G,false> with coef_vec = 0 (c1 column 67, pitch 133) and vec_atomics = 0 (ld_grad_gathered 66);
    # k_bwd_combine<T> over sums with an odd pitch and c1 column
    graph = gpu_csr(P, "zipf", zipf())
    csr = graph[0]
    f = 64
    call = make_call(P, graph, f, dtype, seed=31, aggrs=A6, scalers=S3, bias=True)
    n = csr.n_nodes
    c1col, ldc, ldgg = 67, 133, 66
    coef = torch.full((n, ldc), float("nan"), device=dev())
    gg = torch.zeros((n, ldgg), device=dev())
    gb = torch.full((n, f), float("nan"), device=dev())
    L, lib = call.L, call.lib
    lib.check(L.pna_aggregate_bwd_coef(C.byref(call.d), call.go.data_ptr(), call.go.stride(0), coef.data_ptr(), ldc, c1col,
                                       gg.data_ptr(), ldgg, gb.data_ptr(), f, call.stream()))
    has_in = call.deg > 0
    c0p, c1, gb_closed = B.coef_rows(call.c, call.st, call.deg, np32(call.bias))
    cn = coef.cpu().numpy()
    assert_bits(cn[has_in, :f], c0p[has_in], "c0'")
    assert_bits(cn[has_in, c1col:c1col + f], c1[has_in], "c1")
    assert np.isnan(cn[:, f:c1col]).all() and np.isnan(cn[:, c1col + f:]).all()
    assert_bits(gb.cpu().numpy()[has_in], gb_closed[has_in], "closed-form grad_row_bias")
    # the transposed sums (host restatement), then k_bwd_combine on the device
    rows = np.zeros((n, 2 * f), np.float32)
    rows[:, :f], rows[:, f:] = c0p, c1
    tcsr = csr.transposed(n)
    sums, _ = B.transposed_sums(rows, host_of(tcsr), tcsr.chunk_edges, 2 * f, True)
    lds, sc1 = 2 * f + 5, f + 3
    sbuf = np.full((n, lds), np.nan, np.float32)
    sbuf[:, :f], sbuf[:, sc1:sc1 + f] = sums[:, :f], sums[:, f:]
    sd = torch.from_numpy(sbuf).to(dev())
    lib.check(L.pna_aggregate_bwd_combine(sd.data_ptr(), lds, sc1, call.x.data_ptr(), call.x.stride(0), call.d.dtype, gg.data_ptr(),
                                          ldgg, n, f, call.stream()))
    _check_grad_gathered_coef(call, gg[:, :f].cpu().numpy(), sums[:, :f], sums[:, f:])
    assert (gg[:, f:] == 0).all()


# ---- 8. atomic path end to end ----------------------------------------------------------------------------------------------
def _det(fn):
    torch.use_deterministic_algorithms(True)
    try:
        return fn()
    finally:
        torch.use_deterministic_algorithms(False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_atomic_path_within_the_order_free_bound(P, monkeypatch, dtype):
    # k_bwd_rows<T,VEC,16|8,false> + k_bwd_hub_stats/coef/scatter<...,false>: vector atomics into grad_gathered
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    graph = gpu_csr(P, "zipf", zipf())
    csr = graph[0]
    call = make_call(P, graph, 64, dtype, seed=41, aggrs=A6, scalers=S3, bias=True)
    gg, gb = P.aggregate.aggregate_backward(call.go, call.x, csr, A6, S3, avg_of(csr), row_bias=call.bias, need_bias_grad=True)
    s, bound = B.order_free_sum(csr.n_nodes, call.host[1], call.gm)
    assert B.within_order_free(gg.cpu().numpy(), s, bound).all()
    call.check_bias_atomic(gb.cpu().numpy())


def test_integer_data_is_exact_on_every_path(P, monkeypatch):
    """Integer features and upstream gradients, sum / min / max, identity scaler: every order is exact, so the atomic, the
    coefficient and the deterministic paths must all give the float64 value bit for bit."""
    graph = gpu_csr(P, "zipf", zipf())
    csr = graph[0]
    aggrs = ["sum", "min", "max"]
    call = make_call(P, graph, 32, torch.float32, seed=51, aggrs=aggrs, scalers=["identity"], bias=True, ints=3)
    want = np.zeros((csr.n_nodes, 32))
    np.add.at(want, call.host[1], call.gm.astype(np.float64))
    gb64 = np.zeros((csr.n_nodes, 32))
    np.add.at(gb64, B.slot_rows(call.host[0]), call.gm.astype(np.float64))
    assert np.abs(want).max() > 100            # the probe: sums of many slots, not a trivially small case
    for mode in ("atomic", "coef", "deterministic"):
        monkeypatch.setenv("PNA_B200_BWD", "coef" if mode == "coef" else "atomic")
        run = lambda: P.aggregate.aggregate_backward(call.go, call.x, csr, aggrs, ["identity"], avg_of(csr), row_bias=call.bias,
                                                     need_bias_grad=True)
        gg, gb = _det(run) if mode == "deterministic" else run()
        assert np.array_equal(gg.cpu().numpy().astype(np.float64), want), mode
        assert np.array_equal(gb.cpu().numpy().astype(np.float64), gb64), mode


# ---- 9. deterministic path end to end -----------------------------------------------------------------------------------------
DET_CASES = [
    # F, dtype, bias, slab bytes      instance
    (64, torch.float32, True, None),       # k_bwd_rows<float,4,16,true> + hub chain + k_bwd_hub_bias, then the forward 'sum'
    (128, torch.bfloat16, True, None),     # k_bwd_rows<bf16,8,16,true>
    (75, torch.float32, False, None),      # k_bwd_rows<float,1,32,true>: scalar slots, scalar forward sums
    (128, torch.float32, True, 1 << 20),   # 1 MiB of slots: sixteen feature slabs of 8 columns
]


@pytest.mark.parametrize("f,dtype,bias,slab_bytes", DET_CASES)
def test_deterministic_path_is_exact_for_every_source(P, monkeypatch, f, dtype, bias, slab_bytes):
    graph = gpu_csr(P, "zipf", zipf())
    csr = graph[0]
    call = make_call(P, graph, f, dtype, seed=f + 61, aggrs=A6, scalers=S3, bias=bias)
    tcsr = csr.slot_transposed(csr.n_nodes)
    assert tcsr.n_hubs > 0                      # the probe: heavy sources are split rows of the slot-transposed CSR
    if slab_bytes:
        monkeypatch.setattr(P.aggregate, "DETERMINISTIC_SCRATCH_BYTES", slab_bytes)
    w = P.aggregate.deterministic_slab_width(csr.n_edges, f, 16 // call.x.element_size())
    if slab_bytes:
        assert w < f
    gg, gb = _det(lambda: P.aggregate.aggregate_backward(call.go, call.x, csr, A6, S3, avg_of(csr), row_bias=call.bias,
                                                         need_bias_grad=bias))
    ht = host_of(tcsr)
    want = np.empty((csr.n_nodes, f), np.float32)
    for f0 in range(0, f, w):
        fc = min(w, f - f0)
        vec_ok = fc % 4 == 0 and f % 4 == 0
        want[:, f0:f0 + fc], _ = B.transposed_sums(np.ascontiguousarray(call.gm[:, f0:f0 + fc]), ht, tcsr.chunk_edges, fc, vec_ok)
    assert_bits(gg.cpu().numpy(), want, "deterministic grad_gathered")
    if bias:
        assert_bits(gb.cpu().numpy(), call.gb, "deterministic grad_row_bias")
