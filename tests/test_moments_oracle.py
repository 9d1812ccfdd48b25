"""The moment oracles against the reference's own dense aggregators (tests/golden/dense_moments.pt, k1 = the reference's
aggregate_moment_3/4/5 over dim 2 of X[b, i, j] = h[b, j]): the torch restatement reproduces them, and the C oracle (the
kernel's rounding order) is within the bar of tests/moment_bars.py of float64 and within 2.5x of the reference's own fp32
error."""
import pytest
import torch

from conftest import load_golden
import moment_oracle as MO
import moment_bars as MB


@pytest.fixture(scope="module")
def g():
    return load_golden("dense_moments")


def _edges(adj):
    """adj[b, i, j] != 0  =>  edge (b, j) -> (b, i) over B*N nodes (aggregators.py reduce over dim 2: j is the neighbour)."""
    B, N, _ = adj.shape
    b, i, j = (adj != 0).nonzero(as_tuple=True)
    return j + b * N, i + b * N, B * N


@pytest.mark.parametrize("k", [3, 4, 5])
def test_torch_oracle_reproduces_the_reference(g, k):
    h, adj = g["h"], g["adj"]
    X_j = h.unsqueeze(1).repeat(1, h.size(1), 1, 1)
    got = MO.dense_aggregate_moment(X_j, adj, k)
    torch.testing.assert_close(got, g["k1"][f"moment{k}"], rtol=0, atol=0)


@pytest.mark.parametrize("k", [3, 4, 5])
def test_c_oracle_within_the_bar_and_the_references_own_error(g, k):
    h, adj = g["h"], g["adj"]
    src, dst, n = _edges(adj)
    x = h.reshape(n, -1)
    got = MO.moment(x, torch.stack([src, dst]), n, k)
    r64, tol = MB.moment_bar(x[src], dst, n, k)
    assert ((got.double() - r64).abs() <= tol).all()
    ref32 = g["k1"][f"moment{k}"].reshape(n, -1).double()
    ref_err = float((ref32 - r64).abs().max())
    our_err = float((got.double() - r64).abs().max())
    assert our_err <= 2.5 * ref_err, (our_err, ref_err)
    # the row evaluator the GPU tests use agrees with the reference in float64
    torch.testing.assert_close(MO.moment_rows(x[src].double(), dst, n, k), r64, rtol=1e-12, atol=1e-12)
