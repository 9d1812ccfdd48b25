"""The softmax / softmin / normalised_mean / identity oracles against the reference's own dense aggregators
(tests/golden/dense_weighted.pt, k1 = the reference's functions over dim 2 of X[b, i, j] = h[b, j], with and without
self_loop): the torch restatement reproduces them, and the C oracle (the kernel's rounding order) is within the bar of
tests/weighted_bars.py of float64 and within 2.5x of the reference's own fp32 error."""
import pytest
import torch

from conftest import load_golden
import weighted_oracle as WO
import weighted_bars as WB


@pytest.fixture(scope="module")
def g():
    return load_golden("dense_weighted")


def _edges(adj, self_loop):
    """adj[b, i, j] != 0 (+ I) => edge (b, j) -> (b, i) over B*N nodes, sorted by destination."""
    B, N, _ = adj.shape
    a = adj + torch.eye(N).unsqueeze(0) if self_loop else adj
    b, i, j = (a != 0).nonzero(as_tuple=True)
    return j + b * N, i + b * N, B * N


@pytest.mark.parametrize("self_loop", [False, True])
@pytest.mark.parametrize("name", ["softmax", "softmin", "normalised_mean", "identity"])
def test_torch_oracle_reproduces_the_reference(g, name, self_loop):
    h, adj = g["h"], g["adj"]
    X_j = h.unsqueeze(1).repeat(1, h.size(1), 1, 1)
    got = WO.DENSE[name](X_j, adj, self_loop=self_loop)
    torch.testing.assert_close(got, g["cases"][str(self_loop)]["k1"][name], rtol=0, atol=0)


@pytest.mark.parametrize("self_loop", [False, True])
@pytest.mark.parametrize("name", ["softmax", "softmin", "normalised_mean"])
def test_c_oracle_within_the_bar_and_the_references_own_error(g, name, self_loop):
    h, adj = g["h"], g["adj"]
    src, dst, n = _edges(adj, self_loop)
    x = h.reshape(n, -1)
    got = WO.weighted(x[src], dst, n, name, wsrc=src)
    r64, tol = WB.bar(name, x[src], dst, n, wsrc=src)
    assert ((got.double() - r64).abs() <= tol).all(), float(((got.double() - r64).abs() / tol).max())
    ref32 = g["cases"][str(self_loop)]["k1"][name].reshape(n, -1).double()
    ref_err = float((ref32 - r64).abs().max())
    our_err = float((got.double() - r64).abs().max())
    assert our_err <= 2.5 * ref_err + WB.U * float(r64.abs().max()), (our_err, ref_err)
    # the stable row evaluator the GPU tests use agrees with the reference's formula in float64
    X_j = h.double().unsqueeze(1).repeat(1, h.size(1), 1, 1)
    want = WO.DENSE[name](X_j, adj.double(), self_loop=self_loop).reshape(n, -1)
    torch.testing.assert_close(WO.weighted_rows(x[src].double(), dst, n, name, wsrc=src), want, rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(r64, want, rtol=1e-12, atol=1e-12)
