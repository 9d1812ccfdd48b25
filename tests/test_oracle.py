"""Pin oracle/pna_oracle.py against outputs of the reference's own files (tests/golden, made by oracle/gen_golden.py)."""
import math

import pytest
import torch

from oracle import pna_oracle as O
from conftest import load_golden

SIMPLE = ["pyg_simple_f16", "pyg_simple_f64_hub", "pyg_simple_f75_const", "pyg_simple_allops"]
CONV = ["pyg_conv_t1", "pyg_conv_t4_div", "pyg_conv_t5_rep", "pyg_conv_edge", "pyg_conv_pre2", "pyg_conv_multitask"]

# The fixtures were made on one CPU; the oracle reruns the same torch ops on whatever CPU runs the suite.  Sums, min / max,
# divisions and products are correctly rounded, so the columns built only from them are bit-reproducible on any host.
# torch's vectorised CPU log and sqrt are not correctly rounded and take other code paths on CPUs with other instruction
# sets: the std columns and the log-degree scalers agree to a few ulp.  Matrix products (pre- / post-MLP) are summed in a
# BLAS-dependent order: what passes through them agrees to fp32 GEMM rounding.
FEW_ULP = dict(rtol=1e-6, atol=1e-8)
GEMM_TOL = dict(rtol=1e-5, atol=1e-5)


def assert_aggregate_matches(got, want, aggregators, scalers):
    """[N, S*A*F] aggregate (scaler-major): exact where only correctly rounded operations are involved, FEW_ULP elsewhere."""
    S, A = len(scalers), len(aggregators)
    g, w = got.view(got.size(0), S, A, -1), want.view(want.size(0), S, A, -1)
    for si, sc in enumerate(scalers):
        for ai, ag in enumerate(aggregators):
            if sc in ("amplification", "attenuation") or ag == "std":
                torch.testing.assert_close(g[:, si, ai], w[:, si, ai], **FEW_ULP)
            else:
                assert torch.equal(g[:, si, ai], w[:, si, ai]), (sc, ag)


@pytest.mark.parametrize("name", SIMPLE)
def test_simple_propagate_bit_exact(name):
    g = load_golden(name)
    agg = O.simple_propagate(g["x"], g["edge_index"], g["aggregators"], g["scalers"], g["avg_deg"])
    assert_aggregate_matches(agg, g["aggregate"], g["aggregators"], g["scalers"])    # same torch ops in the same order
    mine = O.avg_deg_from_histogram(g["deg"])
    assert mine["lin"] == g["avg_deg"]["lin"] and mine["log"] == g["avg_deg"]["log"]   # 'exp' overflows to nan for hubs


@pytest.mark.parametrize("name", SIMPLE)
def test_simple_layer_forward(name):
    g = load_golden(name)
    f = g["x"].size(1)
    lay = O.PNAConvSimpleOracle(f, f, g["aggregators"], g["scalers"], g["deg"], post_layers=g["post_layers"])
    lay.load_state_dict(g["state_dict"])
    with torch.no_grad():
        out = lay(g["x"], g["edge_index"])
    torch.testing.assert_close(out, g["out"], **GEMM_TOL)


@pytest.mark.parametrize("name", CONV)
def test_conv_layer_forward(name):
    g = load_golden(name)
    c = g["ctor"]
    lay = O.PNAConvOracle(c["in_channels"], c["out_channels"], g["aggregators"], g["scalers"], g["deg"], edge_dim=c["edge_dim"],
                          towers=c["towers"], pre_layers=c["pre_layers"], post_layers=c["post_layers"],
                          divide_input=c["divide_input"])
    lay.load_state_dict(g["state_dict"])
    x = g["x"]
    xt = x.view(-1, c["towers"], lay.F_in) if c["divide_input"] else x.view(-1, 1, lay.F_in).repeat(1, c["towers"], 1)
    with torch.no_grad():
        agg = lay.propagate(xt, g["edge_index"], g["edge_attr"])
        out = lay(x, g["edge_index"], g["edge_attr"])
    # messages come out of the pre-MLP's matrix products, so the aggregate too agrees to fp32 GEMM rounding -- except that
    # sqrt(var + 1e-5) amplifies that rounding up to 158x where var ~ 0: the std columns are compared through their
    # square, the variance, whose error is fp32 rounding of E[m^2]
    S, A = len(g["scalers"]), len(g["aggregators"])
    std_col = torch.zeros(S, A, agg.size(-1) // (S * A), dtype=torch.bool)
    if "std" in g["aggregators"]:
        std_col[:, g["aggregators"].index("std")] = True
    std_col = std_col.flatten()
    torch.testing.assert_close(agg[..., ~std_col], g["aggregate"][..., ~std_col], **GEMM_TOL)
    torch.testing.assert_close(agg[..., std_col] ** 2, g["aggregate"][..., std_col] ** 2, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(out, g["out"], **GEMM_TOL)


@pytest.mark.parametrize("name", ["dgl_simple", "dgl_simple_var"])
def test_dgl_reduce_matches_reference_mailbox_reduce(name):
    g = load_golden(name)
    ei = g["edge_index"]
    agg = O.dgl_reduce(g["h"][ei[0]], None, ei[1], g["h"].size(0), g["aggregators"].split(), g["scalers"].split(), g["avg_d"])
    assert_aggregate_matches(agg, g["aggregate"], g["aggregators"].split(), g["scalers"].split())
    # in-degree-0 rows are all zero in the DGL flavour, std columns included
    iso = torch.bincount(ei[1], minlength=g["h"].size(0)) == 0
    assert iso.any() and agg[iso].abs().max() == 0
    if "var" in g["aggregators"].split():
        # relu(var) (models/dgl/aggregators.py:22-26): identical neighbour rows give exact zeros, never a negative value
        A = g["aggregators"].split()
        f = g["h"].size(1)
        var_block = agg[:, A.index("var") * f:(A.index("var") + 1) * f]
        assert var_block.min() >= 0 and (var_block[~iso] == 0).any()


def test_dgl_vs_pyg_flavours_differ_only_on_isolated_rows():
    g = load_golden("dgl_simple")
    ei, h = g["edge_index"], g["h"]
    A, S = g["aggregators"].split(), g["scalers"].split()
    d = O.dgl_reduce(h[ei[0]], None, ei[1], h.size(0), A, S, g["avg_d"])
    p = O.simple_propagate(h, ei, A, S, g["avg_d"])
    iso = torch.bincount(ei[1], minlength=h.size(0)) == 0
    torch.testing.assert_close(d[~iso], p[~iso], rtol=2e-6, atol=2e-6)


def test_k1_dense_reference_aggregators():
    """SURVEY 8c K1: the dense reference (imports unmodified) agrees with the scatter restatement."""
    g = load_golden("dense_k1_k2")
    adj, h = g["adj"][0], g["h"][0]
    dst, src = adj.nonzero(as_tuple=True)            # adj[i, j] != 0  =>  edge j -> i
    n = h.size(0)
    msgs = h[src]
    for name in ("mean", "std", "sum", "max", "min"):
        mine = O.AGGREGATORS[name](msgs, dst, n)
        torch.testing.assert_close(mine, g["k1"][name][0], rtol=1e-6, atol=1e-6)
    agg = O.simple_propagate(h, torch.stack([src, dst]), ["mean", "max", "min", "std"],
                             ["identity", "amplification", "attenuation"], g["avg_d"])
    torch.testing.assert_close(agg, g["k1_scaled"][0], rtol=2e-6, atol=2e-6)


def test_k2_numpy_label_reducers():
    """SURVEY 8c K2: float64 numpy neighbourhood reducers of the reference's dataset generator."""
    g = load_golden("dense_k1_k2")
    adj, h = g["adj"][0], g["h"][0]
    dst, src = adj.nonzero(as_tuple=True)
    n = h.size(0)
    msgs = h[src]
    torch.testing.assert_close(O.aggregate_mean(msgs, dst, n).double(), g["k2"]["mean"], rtol=1e-6, atol=1e-6)
    assert torch.equal(O.aggregate_max(msgs, dst, n).double(), g["k2"]["max"])
    assert torch.equal(O.aggregate_min(msgs, dst, n).double(), g["k2"]["min"])
    std_no_eps = torch.sqrt(g["k2"]["std"] ** 2 + 1e-5)
    torch.testing.assert_close(O.aggregate_std(msgs, dst, n).double(), std_no_eps, rtol=1e-5, atol=1e-6)


def test_k3_analytic_rows():
    """in-degree 0: [0, 0, 0, sqrt(1e-5)], amplification -> 0, attenuation -> unchanged; in-degree 1: var == 0."""
    x = torch.tensor([[1.5, -2.0], [0.25, 4.0], [7.0, 7.0]])
    ei = torch.tensor([[0], [1]])                    # single edge 0 -> 1; nodes 0 and 2 isolated
    avg = {"log": 0.7, "lin": 1.3}
    out = O.simple_propagate(x, ei, ["mean", "max", "min", "std"], ["identity", "amplification", "attenuation"], avg)
    e = math.sqrt(1e-5)
    row0 = torch.tensor([0, 0, 0, 0, 0, 0, e, e] + [0] * 8 + [0, 0, 0, 0, 0, 0, e, e], dtype=torch.float32)
    torch.testing.assert_close(out[0], row0, rtol=0, atol=1e-9)
    torch.testing.assert_close(out[2], row0, rtol=0, atol=1e-9)
    amp, att = math.log(2.0) / 0.7, 0.7 / math.log(2.0)
    base = torch.tensor([1.5, -2.0, 1.5, -2.0, 1.5, -2.0, e, e])
    torch.testing.assert_close(out[1], torch.cat([base, base * amp, base * att]), rtol=1e-6, atol=1e-7)


def test_live_reference_over_shims():
    """The reference's own PNAConvSimple.propagate, run over oracle/shims on fresh random inputs and stored by
    oracle/gen_golden.py --live, equals the oracle (bit for bit where the host's CPU kernels allow, see FEW_ULP)."""
    g = load_golden("pyg_simple_live")
    agg = O.simple_propagate(g["x"], g["edge_index"], g["aggregators"], g["scalers"], g["avg_deg"])
    assert_aggregate_matches(agg, g["aggregate"], g["aggregators"], g["scalers"])


def test_c_oracle_agrees_with_torch_oracle():
    """Two independent restatements: torch ops vs scalar C loops in edge order without FMA.  sum / mean / min / max /
    var agree bit for bit (torch's CPU scatter_add_ IS sequential in edge order); sqrt and log differ by <= 1 ulp
    (torch's vectorised CPU sqrt/log are not correctly rounded; glibc's are)."""
    from oracle import c_oracle
    g = torch.Generator().manual_seed(3)
    n, e, f = 400, 5000, 19
    ei = torch.randint(0, n - 40, (2, e), generator=g)
    x = torch.randn(n, f, generator=g)
    A = ["sum", "mean", "min", "max", "var", "std"]
    S = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]
    avg = O.avg_deg_from_histogram(torch.bincount(torch.bincount(ei[1], minlength=n)))
    t = O.simple_propagate(x, ei, A, S, avg)
    c = c_oracle.aggregate(x, ei, A, S, avg)
    assert torch.equal(t[:, :5 * f], c[:, :5 * f])
    torch.testing.assert_close(t, c, rtol=3e-7, atol=1e-9)
    d = O.dgl_reduce(x[ei[0]], None, ei[1], n, ["mean", "max", "min", "std"], S[:3], avg)
    cd = c_oracle.aggregate(x, ei, ["mean", "max", "min", "std"], S[:3], avg, zero_isolated=True)
    torch.testing.assert_close(d, cd, rtol=2e-6, atol=2e-6)


def test_oracles_agree_on_random_ragged_graphs():
    """Property test of the two restatements against each other on ragged inputs: empty graphs, isolated rows, duplicate
    edges, self loops, one-node graphs, a hub, any aggregator / scaler order."""
    from hypothesis import given, settings, strategies as st
    from oracle import c_oracle
    A = ["sum", "mean", "min", "max", "var", "std"]
    S = ["identity", "amplification", "attenuation", "linear", "inverse_linear"]

    @settings(max_examples=40, deadline=None, derandomize=True)
    @given(n=st.integers(1, 40), e=st.integers(0, 300), f=st.integers(1, 9), seed=st.integers(0, 10 ** 6),
           hub=st.booleans(), aggrs=st.permutations(A), scalers=st.permutations(S), na=st.integers(1, 6), ns=st.integers(1, 5))
    def check(n, e, f, seed, hub, aggrs, scalers, na, ns):
        g = torch.Generator().manual_seed(seed)
        ei = torch.randint(0, n, (2, e), generator=g)
        if hub and e:
            ei[1, : e // 2] = 0                                      # half of the edges into one row
        x = torch.randn(n, f, generator=g)
        aggrs, scalers = list(aggrs)[:na], list(scalers)[:ns]
        avg = {"log": 0.5 + float(torch.rand((), generator=g)), "lin": 0.5 + float(torch.rand((), generator=g))}
        t = O.simple_propagate(x, ei, aggrs, scalers, avg)
        c = c_oracle.aggregate(x, ei, aggrs, scalers, avg)
        assert t.shape == c.shape == (n, na * ns * f)
        torch.testing.assert_close(t, c, rtol=3e-6, atol=1e-6)       # sqrt/log: torch's vectorised forms are not correctly rounded
        deg = torch.bincount(ei[1], minlength=n)
        iso = deg == 0
        if bool(iso.any()) and "identity" in scalers and "mean" in aggrs:
            col = (scalers.index("identity") * na + aggrs.index("mean")) * f
            assert torch.equal(c[iso][:, col:col + f], torch.zeros(int(iso.sum()), f))

    check()
