"""Checks of the fp32 restatements in forward_paths_ref.py (CPU only): they equal the plain-C oracle where the kernels'
order is the oracle's, the merge orders are exact on exactly representable data, they are distinguishable on random data,
and the radix-tree walk performs exactly the additions of k_hub_tree."""
import numpy as np
import pytest
import torch

import forward_paths_ref as R
from oracle import c_oracle

ALL_AGGRS = ["sum", "mean", "min", "max", "var", "std"]
SCALERS = ["identity", "linear", "inverse_linear"]
AVG = {"log": 1.7, "lin": 4.3}


def _csr(name, hub_order=None):
    src, dst, n, split, chunk = R.split_graph(name)
    return (src, dst, n, split, chunk) + R.host_csr(src, dst, n, split, chunk, hub_order)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("zero_isolated", [False, True])
def test_restatement_equals_c_oracle_when_every_split_row_is_one_chunk(zero_isolated):
    rng = np.random.default_rng(3)
    n, f = 300, 13
    src, dst = rng.integers(0, n, 2500), rng.integers(0, int(n * 0.85), 2500)
    deg = np.bincount(dst, minlength=n)
    rowptr, col, info, items = R.host_csr(src, dst, n, split=8, chunk=int(deg.max()))
    assert len(info) > 10 and (info[:, 2] == 1).all()
    x = rng.standard_normal((n, f)).astype(np.float32)
    for merge in ("sequential", "two_level", "tree"):
        st = R.row_stats(x, rowptr, col, info, items, int(deg.max()), merge)
        got = R.epilogue(st, deg, ALL_AGGRS, R.host_scales(deg, SCALERS, AVG["log"], AVG["lin"]), zero_isolated=zero_isolated)
        want = c_oracle.aggregate(torch.from_numpy(x), torch.from_numpy(np.stack([src, dst])), ALL_AGGRS, SCALERS, AVG,
                                  zero_isolated=zero_isolated).numpy()
        assert np.array_equal(_bits(got), _bits(want)), merge


def test_light_rows_equal_c_oracle_with_row_bias():
    """Rows below the split threshold, row bias folded in as per-edge messages fl32(x[src] + bias[dst])."""
    rng = np.random.default_rng(4)
    src, dst, n, split, chunk, rowptr, col, info, items = _csr("tree3")
    x = rng.standard_normal((n, 24)).astype(np.float32)
    bias = rng.standard_normal((n, 24)).astype(np.float32)
    deg = np.diff(rowptr)
    st = R.row_stats(x, rowptr, col, info, items, chunk, "tree", bias=bias)
    got = R.epilogue(st, deg, ALL_AGGRS, np.ones((n, 1), np.float32))
    msg = x[src] + bias[dst]                                   # one message row per edge, in edge order
    E = src.size
    pad = np.zeros((max(E, n), 24), np.float32)
    pad[:E] = msg
    want = c_oracle.aggregate(torch.from_numpy(pad), torch.from_numpy(np.stack([np.arange(E), dst])), ALL_AGGRS, ["identity"],
                              AVG).numpy()[:n]
    light = deg < split
    assert light.sum() > 400
    assert np.array_equal(_bits(got[light]), _bits(want[light]))


@pytest.mark.parametrize("name", ["tree3", "edge513", "wide128"])
def test_merge_orders_agree_exactly_on_integer_features(name):
    src, dst, n, split, chunk, rowptr, col, info, items = _csr(name)
    rng = np.random.default_rng(5)
    x = rng.integers(-8, 9, (n, 8)).astype(np.float32)          # every partial sum is an integer below 2^24: exact
    deg = np.diff(rowptr)
    st = {m: R.row_stats(x, rowptr, col, info, items, chunk, m) for m in ("sequential", "two_level", "tree")}
    exact = R.stats_f64(x, rowptr, col)
    for m, s in st.items():
        assert np.array_equal(s.astype(np.float64), exact), m
    outs = [R.epilogue(s, deg, ALL_AGGRS, R.host_scales(deg, SCALERS, 1.7, 4.3)) for s in st.values()]
    assert all(np.array_equal(_bits(o), _bits(outs[0])) for o in outs[1:])
    # past the exact statistics the fp32 epilogue rounds the division and the scale once each (var and std cancel, so the
    # float64 value is no 1-ulp yardstick for them; their inputs were compared exactly above)
    first4 = ["sum", "mean", "min", "max"]
    scales = R.host_scales(deg, SCALERS, 1.7, 4.3)
    np.testing.assert_allclose(R.epilogue(st["tree"], deg, first4, scales),
                               R.epilogue(exact, deg, first4, scales.astype(np.float64)), rtol=2.5e-7, atol=0)


@pytest.mark.parametrize("name", ["tree3", "edge513", "wide128"])
@pytest.mark.parametrize("shuffle", [False, True])
def test_tree_and_two_level_differ_on_random_features(name, shuffle):
    """What lets a bitwise match on the GPU name the merge that ran: the two orders round differently somewhere."""
    src, dst, n, split, chunk = R.split_graph(name)
    n_hubs = int((np.bincount(dst, minlength=n) >= split).sum())
    order = np.random.default_rng(6).permutation(n_hubs) if shuffle else None
    rowptr, col, info, items = R.host_csr(src, dst, n, split, chunk, order)
    assert int(np.diff(rowptr).max()) > R.TREE_MIN_CHUNKS * chunk
    x = np.random.default_rng(7).standard_normal((n, 4)).astype(np.float32)
    tree = R.row_stats(x, rowptr, col, info, items, chunk, "tree")
    two = R.row_stats(x, rowptr, col, info, items, chunk, "two_level")
    assert not np.array_equal(_bits(tree), _bits(two))
    exact = R.stats_f64(x, rowptr, col)
    np.testing.assert_allclose(tree, exact, rtol=1e-4, atol=1e-3)   # both are fp32 sums of the same values
    np.testing.assert_allclose(two, exact, rtol=1e-4, atol=1e-3)


def _layout(*nch):
    """first chunk of the row of every chunk, for rows of nch[0], nch[1], .. chunks laid out in that order"""
    return np.repeat(np.cumsum((0,) + nch[:-1]), nch)


def _expand(rows):
    return [(S, head, pos) for S, head, positions in rows for pos in positions]


def test_tree_walk_hub_starting_mid_block():
    # row A: chunks 0..4, row B: chunks 5..44
    want = _expand([(1, 0, range(1, 5)), (1, 5, range(6, 32)), (1, 32, range(33, 45)),   # level 1: blocks [0,32), [32,64)
                    (32, 5, [32])])                                                         # level 32: B's head keeps 5
    assert R.tree_walk(45, _layout(5, 40)) == want


def test_tree_walk_row_straddling_blocks_at_two_levels():
    # row A: chunks 0..999, row B: chunks 1000..2099
    lvl1 = []
    for base in range(0, 2100, 32):
        for pos in range(base + 1, min(base + 32, 2100)):
            if pos < 1000:
                lvl1.append((1, base, pos))
            elif pos > 1000:
                lvl1.append((1, max(1000, base), pos))
    want = lvl1 + _expand([(32, 0, range(32, 1000, 32)),            # level 32, block [0, 1024): A into 0; 992 is A's
                           (32, 1024, range(1056, 2048, 32)),       # block [1024, 2048): B into the block's base
                           (32, 2048, [2080]),                      # block [2048, 3072)
                           (1024, 1000, [1024, 2048])])             # level 1024: B's two block totals into its head
    assert R.tree_walk(2100, _layout(1000, 1100)) == want


def test_tree_walk_one_chunk_over_rows_beside_a_giant():
    # ten rows of two chunks (0..19), then a row of 50 chunks (20..69)
    want = _expand([(1, 0, [1]), (1, 2, [3]), (1, 4, [5]), (1, 6, [7]), (1, 8, [9]), (1, 10, [11]), (1, 12, [13]),
                    (1, 14, [15]), (1, 16, [17]), (1, 18, [19]), (1, 20, range(21, 32)), (1, 32, range(33, 64)),
                    (1, 64, range(65, 70)), (32, 20, [32, 64])])
    assert R.tree_walk(70, _layout(*([2] * 10), 50)) == want


@pytest.mark.parametrize("nch", [(5, 40), (1000, 1100), tuple([2] * 10) + (50,), (1, 1, 33, 1, 1100, 3)])
def test_tree_totals_equal_the_sequential_merge(nch):
    """On integer partials the walk leaves every row's exact total in its first chunk."""
    first = np.cumsum((0,) + nch[:-1])
    info = np.stack([np.arange(len(nch)), first, np.array(nch), np.array(nch)], 1)
    items = np.concatenate([np.stack([np.full(c, h), np.arange(c)], 1) for h, c in enumerate(nch)])
    P = np.random.default_rng(8).integers(-50, 50, (int(sum(nch)), 4, 3)).astype(np.float32)
    tree = R.merge_tree(P, info, items)
    for h, (f, c) in enumerate(zip(first, nch)):
        assert np.array_equal(tree[h], R.merge_sequential(P, f, c))


def test_lane_group_and_merge_kind():
    assert R.lane_group(16, 4, True) == (4, 1, 1)
    assert R.lane_group(128, 4, True) == (32, 1, 1)
    assert R.lane_group(384, 4, True) == (32, 3, 1)
    assert R.lane_group(1024, 4, True) == (32, 4, 2)
    assert R.lane_group(75, 4, False) == (32, 3, 1)
    assert R.lane_group(2048, 2, True) == (32, 4, 2)
    assert R.merge_kind(512, 1, 32) == "two_level" and R.merge_kind(513, 1, 32) == "tree"
    assert R.merge_kind(513, 1, 16) == "two_level"
