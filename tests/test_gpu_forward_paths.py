"""The forward aggregation's data-selected paths against exact fp32 references (forward_paths_ref.py).

pna_aggregate_fwd picks its kernel instance from the data: row width and alignment (k_rows / k_rows_tiled / k_rows_stream,
lane group G, K, feature blocks), the aggregator / scaler list (Cfg), hot_source_fraction (L1 gathers), partition cost and
residency (dynamic tail), max_degree versus 512 * chunk_edges (radix tree).  Each case below names the instance it is meant
to reach (pna_aggregate_impl.cuh launch_config) and carries a probe that shows the path ran.  Outputs are preallocated
and filled with NaN, so an unwritten row fails.  Rows below the split threshold must equal the slot-order fp32 reduction
of the plain-C oracle bit for bit, split rows the fp32 restatement of the merge that ran; bf16 outputs must equal
round-to-nearest-even bf16 of that fp32 value (one rounding, at the store).  The degree-scaler factors are the kernel's
own (pna_b200.aggregate.row_scales, bit-identical to the epilogue's): one fp32 multiply of the identity block.
"""
import numpy as np
import pytest
import torch

import forward_paths_ref as R

pytestmark = pytest.mark.gpu

A4 = ["mean", "max", "min", "std"]
S3 = ["identity", "amplification", "attenuation"]


@pytest.fixture(scope="module")
def P():
    import pna_b200
    return pna_b200


def dev():
    return torch.device("cuda:0")


def gpu_csr(P, src, dst, n, split=None, chunk=None, n_src=None):
    csr = P.build_csr(torch.from_numpy(np.asarray(src)).to(dev()), torch.from_numpy(np.asarray(dst)).to(dev()), n, split, chunk,
                      n_src=n_src)
    host = (csr.rowptr.cpu().numpy().astype(np.int64), csr.col.cpu().numpy().astype(np.int64),
            csr.hub_info.cpu().numpy().astype(np.int64).reshape(-1, 4), csr.chunk_items.cpu().numpy().astype(np.int64).reshape(-1, 2))
    return csr, host


def avg_of(csr):
    deg = csr.in_degree.long().cpu()
    hist = torch.bincount(deg).double()
    b = torch.arange(hist.numel(), dtype=torch.float64)
    return {"log": float(((b + 1).log() * hist).sum() / hist.sum()), "lin": float((b * hist).sum() / hist.sum())}


def run(P, x, csr, aggrs, scalers, avg, towers=1, self_feat=None, **kw):
    width = towers * ((self_feat is not None) + len(aggrs) * len(scalers)) * (x.size(1) // towers)
    out = torch.full((csr.n_nodes, width), float("nan"), dtype=x.dtype, device=dev())
    P.aggregate_forward(x, csr, aggrs, scalers, avg, towers=towers, self_feat=self_feat, out=out, **kw)
    return out


def np32(t):
    return t.float().cpu().numpy()


def reference(P, x, csr, host, aggrs, scalers, avg, merge, bias=None, towers=1, self_feat=None, **epi):
    """fp32 reference of aggregate_forward(x, ...) on the CSR as built (the tree walks the GPU's own chunk layout)."""
    rowptr, col, info, items = host
    st = R.row_stats(np32(x), rowptr, col, info, items, csr.chunk_edges, merge, None if bias is None else np32(bias))
    scales = P.aggregate.row_scales(csr, scalers, avg).cpu().numpy()
    return R.epilogue(st, np.diff(rowptr), aggrs, scales, towers=towers, self_feat=None if self_feat is None else np32(self_feat),
                      **epi)


def bits(t, dtype):
    """integer view of a result in `dtype` (fp32 reference values are rounded to bf16 once, to nearest even)"""
    t = torch.as_tensor(t).cpu().to(dtype)
    return t.view(torch.int16 if dtype == torch.bfloat16 else torch.int32)


def assert_bits(got, want, rows=None):
    g = bits(got, got.dtype)
    w = bits(want, got.dtype)
    if rows is not None:
        g, w = g[rows], w[rows]
    bad = (g != w).any(1).nonzero().flatten()
    assert bad.numel() == 0, f"{bad.numel()} rows differ, first {bad[:8].tolist()}"


def features(n, f, dtype, seed, layout="contig"):
    """[n, f] on the GPU; layout "pitch+2" = view of an [n, f+2] buffer (odd pitch, scalar path), "offset1" = columns
    1..f of an [n, f+4] buffer (misaligned base, scalar path)."""
    g = torch.Generator().manual_seed(seed)
    if layout == "contig":
        return torch.randn(n, f, generator=g).to(dtype).to(dev())
    if layout == "pitch+2":
        return torch.randn(n, f + 2, generator=g).to(dtype).to(dev())[:, :f]
    return torch.randn(n, f + 4, generator=g).to(dtype).to(dev())[:, 1:1 + f]


# ---- 1. split rows: radix tree (k_hub_tree) versus the two-level merge ------------------------------------------------
TREE_CASES = [
    # graph, F, dtype, layout, options                         instance (launch_config)
    ("tree3", 128, torch.float32, "contig", {}),              # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,BIAS=0>, chunk pseudo-rows, k_hub_tree x3 levels
    ("tree3", 256, torch.float32, "contig", {}),              # k_rows_stream<float,4,K=2,...>, tree
    ("tree3", 384, torch.float32, "contig", {}),              # k_rows_stream<float,4,K=3,...>, tree
    ("tree3", 512, torch.float32, "contig", {}),              # k_rows_stream<float,4,K=4,...>, tree
    ("tree3", 1024, torch.float32, "contig", {}),             # k_rows_stream<float,4,K=4>, gridDim.y = 2, tree per feature block
    ("tree3", 75, torch.float32, "pitch+2", {}),              # k_rows_tiled<float,1,G=32,K=3,U=2,CfgMeanMaxMinStd,0> + k_hub_chunks, tree
    ("tree3", 256, torch.bfloat16, "contig", {}),             # k_rows_stream<bf16,8,K=1,CfgMeanMaxMinStd,0>, tree
    ("tree3", 2048, torch.bfloat16, "contig", {}),            # k_rows_stream<bf16,8,K=4>, gridDim.y = 2, tree
    ("tree3", 256, torch.float32, "contig", {"bias": True}),  # k_rows_stream<float,4,K=2,CfgMeanMaxMinStd,BIAS=1>, tree
    ("tree3", 75, torch.float32, "pitch+2", {"bias": True}),  # k_rows_tiled<float,1,32,3,2,CfgMeanMaxMinStd,BIAS=1> + k_hub_chunks (bias), tree
    ("tree3", 256, torch.bfloat16, "contig", {"bias": True}),  # k_rows_stream<bf16,8,K=1,CfgMeanMaxMinStd,BIAS=1>, tree
    ("tree3", 256, torch.float32, "contig", {"towers": 2}),   # k_rows_stream<float,4,K=2,CfgMeanMaxMinStd>, 2 towers + self block, tree
    ("tree3", 128, torch.float32, "contig", {"dynamic": True}),  # k_rows_stream<float,4,K=1,CfgDynamic,0>, tree
    ("tree3", 16, torch.float32, "contig", {}),               # k_rows_tiled<float,4,G=4,K=1> + k_hub_chunks + two-level k_hub_finalize (G < 32)
    ("edge512", 128, torch.float32, "contig", {}),            # k_rows_stream<float,4,K=1>, max_degree == 512 * chunk: two-level
    ("edge513", 128, torch.float32, "contig", {}),            # k_rows_stream<float,4,K=1>, max_degree == 512 * chunk + 1: tree
    ("edge513", 75, torch.float32, "pitch+2", {}),            # k_rows_tiled<float,1,32,3,2> + k_hub_chunks, tree
    ("wide128", 128, torch.float32, "contig", {}),            # k_rows_stream<float,4,K=1>, 128-slot chunks, 520-chunk row, tree
    ("wide128", 1024, torch.float32, "contig", {}),           # k_rows_stream<float,4,K=4>, gridDim.y = 2, tree
]

_GRAPHS = {}


def split_case_graph(P, name):
    if name not in _GRAPHS:
        src, dst, n, split, chunk = R.split_graph(name)
        _GRAPHS[name] = gpu_csr(P, src, dst, n, split, chunk)
    return _GRAPHS[name]


def _tree_blocks_are_straddled(info, n_chunks):
    """probe of the layout: at levels 1 and 32 some split row starts mid-block and continues into the next block"""
    firsts, ends = info[:, 1], info[:, 1] + info[:, 2]
    for S in (1, 32):
        blk = R.TREE_R * S
        if not ((firsts % blk != 0) & (firsts // blk < (ends - 1) // blk)).any():
            return False
    return n_chunks > R.TREE_R ** 2


@pytest.mark.parametrize("name,f,dtype,layout,opt", TREE_CASES)
def test_split_rows_merge_as_launch_config_chooses(P, name, f, dtype, layout, opt):
    csr, host = split_case_graph(P, name)
    n = csr.n_nodes
    x = features(n, f, dtype, seed=f, layout=layout)
    aggrs, scalers = (["sum", "var", "max"], ["linear", "inverse_linear"]) if opt.get("dynamic") else (A4, S3)
    avg = avg_of(csr)
    kw, ekw = {}, {}
    if opt.get("bias"):
        kw["row_bias"] = features(n, f, dtype, seed=f + 1)
    if opt.get("towers"):
        kw.update(towers=2, self_feat=features(n, f, dtype, seed=f + 2))
        ekw.update(towers=2, self_feat=kw["self_feat"])
    G = R.lane_group(f, x.element_size(), layout == "contig")[0]
    merge = R.merge_kind(csr.max_degree, csr.chunk_edges, G)
    assert merge == ("two_level" if (name == "edge512" or f == 16) else "tree")
    got = run(P, x, csr, aggrs, scalers, avg, **kw)
    split_rows = host[2][:, 0]
    tree = reference(P, x, csr, host, aggrs, scalers, avg, "tree", bias=kw.get("row_bias"), **ekw)
    two = reference(P, x, csr, host, aggrs, scalers, avg, "two_level", bias=kw.get("row_bias"), **ekw)
    # the probe: the two merges round differently on these rows, so matching one of them names the merge that ran (in fp32:
    # one bf16 rounding of 41 rows can hide every difference)
    assert not np.array_equal(tree[split_rows], two[split_rows])
    assert_bits(got, tree if merge == "tree" else two)
    if name == "tree3" and merge == "tree":
        assert _tree_blocks_are_straddled(host[2], csr.n_chunks)


def test_folded_finalize_is_off_with_the_tree(P, monkeypatch):
    """PNA_B200_FOLD_FINALIZE=1 with the tree: the same bits, and the completion counters are never touched."""
    csr, host = split_case_graph(P, "tree3")
    x = features(csr.n_nodes, 128, torch.float32, seed=3)
    avg = avg_of(csr)
    monkeypatch.setenv("PNA_B200_FOLD_FINALIZE", "1")
    got = run(P, x, csr, A4, S3, avg)       # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,FOLD=0> + k_hub_tree
    assert_bits(got, reference(P, x, csr, host, A4, S3, avg, "tree"))
    assert int(csr.hub_done().abs().sum()) == 0


# ---- 2. dynamic tail of the streamed kernel (pna_agg_t.work_counter) --------------------------------------------------
SENTINEL = -12345


@pytest.fixture(scope="module")
def tail(P):
    src, dst, n = R.tail_graph()
    csr, host = gpu_csr(P, src, dst, n)
    assert csr.n_hubs >= 8 and csr.n_part == 65536
    return csr, host


def _run_counted(P, monkeypatch, on, *args, **kw):
    csr = args[1]
    monkeypatch.setattr(P.aggregate, "DYNAMIC_TAIL_MIN_PARTITION_COST", 0 if on else 1 << 40)
    csr.work_counter().fill_(SENTINEL)
    out = run(P, *args, **kw)
    return out, int(csr.work_counter().item())


def _assert_blockwise(P, got, x, csr, host, aggrs, scalers, avg, bias=None, **epi):
    """reference in row blocks (the [N, 4, F] statistics once, the epilogue per block) to bound host memory"""
    rowptr, col, info, items = host
    st = R.row_stats(np32(x), rowptr, col, info, items, csr.chunk_edges, "two_level", None if bias is None else np32(bias))
    scales = P.aggregate.row_scales(csr, scalers, avg).cpu().numpy()
    deg = np.diff(rowptr)
    for r0 in range(0, csr.n_nodes, 1 << 15):
        sl = slice(r0, r0 + (1 << 15))
        assert_bits(got[sl], R.epilogue(st[sl], deg[sl], aggrs, scales[sl], **epi))


TAIL_CASES = [
    # F, dtype, aggregators, scalers, options                   instance (launch_config), all with the dynamic tail
    (128, torch.float32, A4, S3, {}),                            # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,BIAS=0,FOLD=0>
    (128, torch.float32, A4, ["identity"], {}),                  # k_rows_stream<float,4,K=1,CfgMeanMaxMinStdId,0,0>
    (128, torch.float32, ["sum", "var", "max"], ["linear", "inverse_linear"], {}),   # k_rows_stream<...,CfgDynamic,0,0>
    (128, torch.float32, A4, S3, {"bias": True}),                # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,BIAS=1,0>
    (128, torch.float32, A4, S3, {"fold": True}),                # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,0,FOLD=1>
    (128, torch.float32, A4, S3, {"l1": True}),                  # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,0,0,L1=1>
    (256, torch.bfloat16, A4, ["identity"], {}),                 # k_rows_stream<bf16,8,K=1,CfgMeanMaxMinStdId,0,0>
]


@pytest.mark.parametrize("f,dtype,aggrs,scalers,opt", TAIL_CASES)
def test_dynamic_tail_hands_out_every_partition_once(P, tail, monkeypatch, f, dtype, aggrs, scalers, opt):
    csr, host = tail
    x = features(csr.n_nodes, f, dtype, seed=40 + f)
    avg = avg_of(csr)
    kw = {}
    if opt.get("bias"):
        kw["row_bias"] = features(csr.n_nodes, f, dtype, seed=41)
    if opt.get("l1"):
        kw["gather_l1"] = True
    monkeypatch.setenv("PNA_B200_FOLD_FINALIZE", "1" if opt.get("fold") else "0")
    on, ctr_on = _run_counted(P, monkeypatch, True, x, csr, aggrs, scalers, avg, **kw)
    off, ctr_off = _run_counted(P, monkeypatch, False, x, csr, aggrs, scalers, avg, **kw)
    # each of the n_part - n_static dynamic partitions handed out once, plus one failed grab per warp (W warps)
    n_static = csr.n_part * 7 // 10
    W = ctr_on - (csr.n_part - n_static)
    sms = torch.cuda.get_device_properties(dev()).multi_processor_count
    assert W > 0 and W % (4 * sms) == 0, (ctr_on, W, sms)
    assert ctr_off == SENTINEL
    assert_bits(on, off)
    _assert_blockwise(P, on, x, csr, host, aggrs, scalers, avg, bias=kw.get("row_bias"))
    if opt.get("fold"):
        assert int(csr.hub_done().abs().sum()) == 0


def test_dynamic_tail_is_dropped_with_several_feature_blocks(P, tail, monkeypatch):
    csr, host = tail
    x = features(csr.n_nodes, 1024, torch.float32, seed=50)
    avg = avg_of(csr)
    # k_rows_stream<float,4,K=4,CfgDynamic>, gridDim.y = 2: the launcher clears work_counter
    on, ctr = _run_counted(P, monkeypatch, True, x, csr, ["sum"], ["identity"], avg)
    assert ctr == SENTINEL
    off, _ = _run_counted(P, monkeypatch, False, x, csr, ["sum"], ["identity"], avg)
    assert_bits(on, off)


# ---- 3. L1 gathers (PNA_FLAG_GATHER_L1) ------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hot(P):
    from pna_b200 import synth
    ei, _ = synth.powerlaw(n_nodes=40_000, n_edges=400_000, n_feat=1, seed=3, with_features=False)
    csr, host = gpu_csr(P, ei[0].numpy(), ei[1].numpy(), 40_000)
    assert csr.hot_source_fraction > P.aggregate.HOT_SOURCE_FRACTION_FOR_L1     # auto-selection takes the L1 path
    return ei, csr, host


L1_CASES = [
    # scalers, bias      instance with gather_l1 (launch_config)
    (S3, False),         # k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,0,1,FOLD=0,L1=1>
    (["identity"], False),   # k_rows_stream<float,4,K=1,CfgMeanMaxMinStdId,0,1,FOLD=0,L1=1>
    (S3, True),          # row bias: no L1 instance -> k_rows_stream<float,4,K=1,CfgMeanMaxMinStd,BIAS=1>
    (["identity"], True),    # row bias: no L1 instance -> k_rows_stream<float,4,K=1,CfgDynamic,BIAS=1>
]


@pytest.mark.parametrize("scalers,bias", L1_CASES)
def test_l1_gathers_are_bit_identical(P, hot, scalers, bias):
    _, csr, host = hot
    n, f = csr.n_nodes, 128
    x = features(n, f, torch.float32, seed=60)
    avg = avg_of(csr)
    kw = {"row_bias": features(n, f, torch.float32, seed=61)} if bias else {}
    auto = run(P, x, csr, A4, scalers, avg, **kw)
    l1 = run(P, x, csr, A4, scalers, avg, gather_l1=True, **kw)
    plain = run(P, x, csr, A4, scalers, avg, gather_l1=False, **kw)
    merge = R.merge_kind(csr.max_degree, csr.chunk_edges, 32)
    want = reference(P, x, csr, host, A4, scalers, avg, merge, bias=kw.get("row_bias"))
    for got in (auto, l1, plain):
        assert_bits(got, want)


def test_compact_layer_on_a_hot_source_graph(P, hot):
    """PNAConvSimple's compact post path (identity-scaled aggregate, L1 instance CfgMeanMaxMinStdId) against the oracle.
    The post linear is a dot product of K = 12 * 96 = 1152 fp32 terms: the bar is that of test_gpu_parity.py
    test_layer_output_error_at_config2_width, the forward error of a dot product against the size of what it sums."""
    from oracle import pna_oracle as O
    ei, csr, _ = hot
    n, f = csr.n_nodes, 96                       # the narrowest fp32 width of the streamed kernel that keeps K small
    x = torch.randn(n, f, generator=torch.Generator().manual_seed(62))
    deg = torch.bincount(torch.bincount(ei[1], minlength=n))
    torch.manual_seed(63)
    ref = O.PNAConvSimpleOracle(f, 128, A4, S3, deg)
    lay = P.PNAConvSimple(f, 128, A4, S3, deg)
    lay.load_state_dict(ref.state_dict())
    lay = lay.to(dev())
    xd = x.to(dev())
    assert lay._compact(xd)
    with torch.no_grad():
        got = lay(xd, ei.to(dev()), csr=csr).cpu().double()
        want32 = ref(x, ei).double()
        agg64 = O.simple_propagate(x.double(), ei, A4, S3, ref.avg_deg)
        W, b = ref.post_nn[0].weight.double(), ref.post_nn[0].bias.double()
        want64 = agg64 @ W.t() + b
        cond = agg64.abs() @ W.abs().t() + b.abs()
    err_gpu = float(((got - want64).abs() / cond).max())
    err_ref = float(((want32 - want64).abs() / cond).max())
    assert err_gpu <= 1e-5, (err_gpu, err_ref)


# ---- 4 + 5. CfgDynamic on every kernel family; bf16 is one rounding of the fp32 value ------------------------------------
@pytest.fixture(scope="module")
def small(P):
    rng = np.random.default_rng(70)
    src, dst = R._with_rows(rng, 400, 3000, 0, {397: 700, 398: 1500})      # 6 chunks (sequential), 12 (two-level)
    dst[rng.random(dst.size) < 0.1] = 399                                  # ... and a third split row
    dst = np.where(dst < 30, 31, dst)                                      # rows 0..29 isolated
    return gpu_csr(P, src, dst, 400)


DYN = [  # aggregators, scalers, flags
    (["sum", "var"], ["linear", "inverse_linear"], {"relu_var": True}),
    (["std", "min", "mean"], ["identity", "attenuation"], {"zero_isolated": True}),
    (["max"], ["amplification"], {}),
    (["var", "sum", "max", "min", "mean", "std"], ["inverse_linear", "identity", "linear", "attenuation", "amplification"], {}),
]
WIDTHS = [
    # F, dtype, layout          instance (launch_typed / launch_config), all CfgDynamic
    (1, torch.float32, "contig"),      # scalar, G=1: k_rows<float,1,1,1,4,CfgDynamic>
    (3, torch.float32, "contig"),      # scalar, G=4: k_rows_tiled<float,1,4,1,4,CfgDynamic,0>
    (4, torch.float32, "contig"),      # VEC=4, G=1: k_rows<float,4,1,1,4>
    (8, torch.float32, "contig"),      # G=2: k_rows<float,4,2,1,4>
    (16, torch.float32, "contig"),     # G=4: k_rows_tiled<float,4,4,1,4>
    (32, torch.float32, "contig"),     # G=8: k_rows_tiled<float,4,8,1,4>
    (64, torch.float32, "contig"),     # G=16: k_rows_tiled<float,4,16,1,4>
    (128, torch.float32, "contig"),    # k_rows_stream<float,4,K=1,CfgDynamic,0>
    (256, torch.float32, "contig"),    # k_rows_stream<float,4,K=2>
    (384, torch.float32, "contig"),    # k_rows_stream<float,4,K=3>
    (512, torch.float32, "contig"),    # k_rows_stream<float,4,K=4>
    (1024, torch.float32, "contig"),   # k_rows_stream<float,4,K=4>, gridDim.y = 2
    (1536, torch.float32, "contig"),   # k_rows_stream<float,4,K=4>, gridDim.y = 3
    (37, torch.float32, "offset1"),    # misaligned scalar, G=32: k_rows_tiled<float,1,32,2,2>
    (75, torch.float32, "pitch+2"),    # odd pitch scalar, G=32: k_rows_tiled<float,1,32,3,2>
    (8, torch.bfloat16, "contig"),     # VEC=8, G=1: k_rows<bf16,8,1,1,4>
    (64, torch.bfloat16, "contig"),    # G=8: k_rows_tiled<bf16,8,8,1,4>
    (256, torch.bfloat16, "contig"),   # k_rows_stream<bf16,8,K=1>
    (512, torch.bfloat16, "contig"),   # k_rows_stream<bf16,8,K=2>
    (768, torch.bfloat16, "contig"),   # k_rows_stream<bf16,8,K=3>
    (1024, torch.bfloat16, "contig"),  # k_rows_stream<bf16,8,K=4>
    (2048, torch.bfloat16, "contig"),  # k_rows_stream<bf16,8,K=4>, gridDim.y = 2
    (50, torch.bfloat16, "offset1"),   # misaligned bf16 scalar, G=32: k_rows_tiled<bf16,1,32,2,2>
]


@pytest.mark.parametrize("f,dtype,layout", WIDTHS)
def test_dynamic_lists_on_every_kernel_family(P, small, f, dtype, layout):
    csr, host = small
    x = features(csr.n_nodes, f, dtype, seed=80 + f, layout=layout)
    avg = avg_of(csr)
    for aggrs, scalers, flags in DYN:
        got = run(P, x, csr, aggrs, scalers, avg, **flags)
        assert_bits(got, reference(P, x, csr, host, aggrs, scalers, avg, "two_level", **flags))


# ---- 6. rows more than 4 GiB past the start of the gathered buffer -----------------------------------------------------
def any_nonzero(t):
    """in row slices: a whole-tensor count_nonzero of a 4.5 GB gradient allocates twice its size"""
    return any(bool(t[r0:r0 + (1 << 17)].any()) for r0 in range(0, t.size(0), 1 << 17))


def test_rows_past_4_gib(P, monkeypatch):
    free, _ = torch.cuda.mem_get_info(dev())
    if free < 16 * 2 ** 30:
        pytest.skip(f"needs 16 GiB of free device memory for a 4.5 GB gathered buffer and its gradient, {free / 2 ** 30:.1f} free")
    from pna_b200 import synth
    from pna_b200.aggregate import aggregate_backward
    F, N, n_src = 1024, 20_000, 1_100_000
    rng = np.random.default_rng(90)
    deg = rng.integers(0, 15, N)
    deg[17] = 1000                                                       # one split row (default threshold 256)
    dst = np.repeat(np.arange(N), deg)
    far = rng.random(dst.size) < 0.8                                     # 80 % of the sources at byte offsets >= 4 GiB
    src = np.where(far, rng.integers(1 << 20, n_src, dst.size), rng.integers(0, 1 << 20, dst.size))
    uniq, src_c = np.unique(src, return_inverse=True)
    big, big_host = gpu_csr(P, src, dst, N, n_src=n_src)
    comp, _ = gpu_csr(P, src_c, dst, N, n_src=uniq.size)
    assert big.n_hubs == 1 and np.array_equal(big_host[1], uniq[comp.col.cpu().numpy()])   # same slot order
    x_big = torch.empty((n_src, F), dtype=torch.float32, device=dev())
    for r0 in range(0, n_src, 1 << 16):                                  # filled in slices: bounded temporaries
        r1 = min(n_src, r0 + (1 << 16))
        x_big[r0:r1] = synth.hash_features(torch.arange(r0, r1, device=dev()), F, chunk=1 << 14)
    u = torch.from_numpy(uniq).to(dev())
    x_c = synth.hash_features(u, F, chunk=1 << 14)
    avg = avg_of(big)
    views = [(slice(None), "k_rows_stream<float,4,K=4>, gridDim.y = 2; addresses formed in issue_half"),
             (slice(0, 256), "k_rows_stream<float,4,K=2>, 4 KB pitch"),
             (slice(0, 64), "k_rows_tiled<float,4,G=16,K=1>; addresses formed in local_row"),
             (slice(1, 76), "k_rows_tiled<float,1,G=32,K=3>, misaligned")]
    for cols, what in views:
        got = run(P, x_big[:, cols], big, A4, S3, avg)
        want = run(P, x_c[:, cols], comp, A4, S3, avg)
        assert not bool(got.isnan().any()) and torch.equal(got.view(torch.int32), want.view(torch.int32)), what
        del got, want
    # backward at full width: the deterministic path writes grad rows through the forward kernel's `out`
    go = torch.randn(N, 12 * F, generator=torch.Generator(device=dev()).manual_seed(91), device=dev())
    torch.use_deterministic_algorithms(True)
    try:
        g_big, _ = aggregate_backward(go, x_big, big, A4, S3, avg)
        g_c, _ = aggregate_backward(go, x_c, comp, A4, S3, avg)
    finally:
        torch.use_deterministic_algorithms(False)
    det = g_big[u]
    assert torch.equal(det.view(torch.int32), g_c.view(torch.int32))
    del g_c
    g_big[u] = 0
    assert not any_nonzero(g_big)                                        # rows nobody gathers get no gradient
    del g_big
    monkeypatch.setenv("PNA_B200_BWD", "atomic")
    g_at, _ = aggregate_backward(go, x_big, big, A4, S3, avg)
    scale = float(det.abs().max())
    assert float((g_at[u] - det).abs().max()) <= 1e-6 * scale           # per-edge atomics: only the summation order differs
    g_at[u] = 0
    assert not any_nonzero(g_at)
    del g_at, det, go, x_big, x_c
    torch.cuda.empty_cache()
